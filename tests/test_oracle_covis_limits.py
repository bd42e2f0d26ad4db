"""CPU test of the scenes of tests/covis_limit_scenes.py: each reaches the size it is built for (counter entries, events per
target, touched slots per batch, map and list lengths, observation list lengths, candidates, n0), read from the scene's
model and from the oracle; and on each the oracle equals the reference's own KeyFrame.cc, MapPoint.cc, LocalMapping.cc and
Tracking.cc, through the run() helpers of test_oracle_covis.py, test_oracle_observations.py, test_oracle_kf_culling.py and
test_oracle_local_map.py (touched keyframes only where a full compare after every step is too slow)."""
import copy

import numpy as np
import pytest

import covis_limit_scenes as L
import covis_scenes as S
import observation_scenes as OS
import test_oracle_covis as TC
import test_oracle_kf_culling as TK
import test_oracle_local_map as TL
import test_oracle_observations as TO
from oracle import covis as OC
from oracle import kf_culling as KC
from oracle import local_map as LM
from oracle import observations as OO
from oracle.covis import CovisOracle

needs_ref = pytest.mark.skipif(not OC.ref_available(), reason="oracle/_ref/libref_drivers.so not built (needs the reference sources)")
needs_cull = pytest.mark.skipif(not KC.ref_available(), reason="oracle/_ref/libref_kf_culling.so not built (needs the reference sources)")
needs_lm = pytest.mark.skipif(not LM.ref_available(), reason="oracle/_ref/libref_local_map.so not built (needs the reference sources)")

GRAPH = L.counter_scenes() + L.capacity_scenes() + L.batch_scenes() + L.erase_scenes()


def counter(model, kf):
    """KFcounter of UpdateConnections: one count per row cell whose point is not bad, per other observer"""
    c = {}
    for m in model.kf_mp[kf, :model.nfeat[kf]].tolist():
        if m < 0 or model.bad[m]:
            continue
        for k in model.obs[m]:
            if k != kf:
                c[k] = c.get(k, 0) + 1
    return c


def filtered(c, model):
    """the AddConnection targets of one call: weights >= 15, else the first maximum in key order"""
    if not c:
        return []
    t = [k for k, w in c.items() if w >= 15]
    if t:
        return t
    top = max(c.values())
    return [min((k for k, w in c.items() if w == top), key=model.key)]


def batch_sizes(scene):
    """per update step: (batch, counter sizes, events per target, touched slots), from the model alone"""
    model, out = S.Model(scene, scene.keys), []
    for step in scene.steps + ([("update", scene.refused)] if scene.refused else []):
        model.apply(step)
        if step[0] != "update":
            continue
        ev, touched, sizes = {}, set(step[1]), []
        for kf in step[1]:
            c = counter(model, kf)
            sizes.append(len(c))
            for t in filtered(c, model):
                ev[t] = ev.get(t, 0) + 1
                touched.add(t)
        out.append(dict(batch=list(step[1]), sizes=sizes, events=ev, touched=len(touched)))
    return out


def oracle_maps(scene, upto=None):
    """the oracle's graph after the scene's steps (and its refused batch, which the oracle has no bound for)"""
    model, slot_of = S.Model(scene, scene.keys), scene.slots()
    orc = CovisOracle(scene.nkf)
    steps = scene.steps + ([("update", scene.refused)] if scene.refused else [])
    for k in range(scene.nkf):
        orc.add(slot_of[k], k, int(k if scene.keys is None else scene.keys[k]))
    for step in steps[:upto]:
        model.apply(step)
        if step[0] == "update":
            kf_mp, counts, gp, obs = model.inputs(slot_of, scene.nkf)
            orc.replay([int(slot_of[k]) for k in step[1]], kf_mp, counts, scene.cap, gp, obs)
        elif step[0] == "erase_kf":
            orc.erase(slot_of[step[1]])
    return orc, slot_of


def test_counter_scenes_reach_their_sizes():
    for s in L.counter_scenes():
        b = batch_sizes(s)
        f = s.facts
        assert b[0]["sizes"] == [f["counter"]], s.name
        orc, slot_of = oracle_maps(s, upto=next(i for i, st in enumerate(s.steps) if st[0] == "update") + 1)
        hub = int(slot_of[f["hub"]])
        assert len(orc.weights(hub)[0]) == f["counter"] and len(orc.ordered(hub)[0]) == f["filtered"], s.name
        ws = sorted(set(f["weights"]))
        assert ws == ([12, 13, 14] if "below" in s.name else [14, 15, 16]), s.name
        if "below" in s.name:   # the first maximum: the smallest key among ~n/3 tied leaves, neither the first slot nor the oldest
            tied = [k for k, w in zip(range(2, f["counter"] + 2), f["weights"]) if w == 14]
            first = min(tied, key=lambda k: int(s.keys[k]))
            assert len(tied) > 300 and orc.ordered(hub)[0] == [int(slot_of[first])]
            assert first != min(tied) and int(slot_of[first]) != min(int(slot_of[k]) for k in tied)
        orc.close()
    # the count kernel's block is 512 and the apply / erase blocks 256: every size past them, with one thread per entry
    # below them as control
    assert {s.facts["counter"] for s in L.counter_scenes()} >= {511, 512, 513, 1024, 1025, 2047, 2048}


def test_capacity_scenes_reach_their_sizes():
    for s in L.capacity_scenes():
        b = batch_sizes(s)
        f = s.facts
        if s.name.startswith("target_full"):
            assert b[0]["sizes"] == [f["C"]] and b[-1]["events"] == {f["target"]: 1}, s.name
            orc, slot_of = oracle_maps(s)
            assert len(orc.weights(int(slot_of[f["target"]]))[0]) == f["C"] + 1   # one past max_connections
            orc.close()
            continue
        hub_batch = next(x for x in b if x["batch"] == [f["hub"]])
        assert hub_batch["sizes"] == [f["counter"]], s.name
        assert (f["counter"] > f["C"]) == (s.refused is not None), s.name
        assert f["full"] == (f["counter"] > f["P"]), s.name
    full = {(s.facts["C"], s.facts["counter"]) for s in L.capacity_scenes() if s.facts.get("full")}
    assert full == {(6, 17), (2048, 4097)}


def test_batch_scenes_reach_their_sizes():
    hub1024, hub1000, wide = L.batch_scenes()
    for s in (hub1024, hub1000):
        b = batch_sizes(s)
        hub = s.facts["hub"]
        assert len(b[0]["batch"]) == len(b[1]["batch"]) == s.facts["batch"]
        assert b[0]["events"][hub] == s.facts["batch"]            # every entry sends the hub an event: E holds all of them
        assert hub not in b[0]["batch"] and b[1]["batch"].index(hub) == s.facts["own_at"]
        after = sum(1 for k in b[1]["batch"][s.facts["own_at"] + 1:] if k != hub)
        assert after == s.facts["events"][1] > 256                 # the events applied after the hub's own call
    b = batch_sizes(wide)
    assert [x["touched"] for x in b] == [wide.facts["touched"]] * 2 and wide.facts["touched"] > 1024


def test_erase_scenes_reach_their_sizes():
    hub_s, leaf_s = L.erase_scenes()
    orc, slot_of = oracle_maps(hub_s, upto=[i for i, st in enumerate(hub_s.steps) if st[0] == "update"][0] + 1)
    hub = int(slot_of[hub_s.facts["hub"]])
    assert len(orc.weights(hub)[0]) == 2048 and all(hub in orc.weights(int(slot_of[k]))[0] for k in range(2, 2050))
    orc.close()
    erase_at = [i for i, st in enumerate(leaf_s.steps) if st[0] == "erase_kf"]
    orc, slot_of = oracle_maps(leaf_s, upto=erase_at[0])
    hub, named, stale = (int(slot_of[leaf_s.facts[k]]) for k in ("hub", "named", "stale"))
    assert len(orc.weights(hub)[0]) == 2048 and named in orc.weights(hub)[0] and stale in orc.weights(hub)[0]
    assert hub in orc.weights(named)[0] and orc.weights(stale)[0] == [int(slot_of[0])]   # the stale leaf's map: keyframe 0 only
    orc.close()
    orc, slot_of = oracle_maps(leaf_s, upto=erase_at[1] + 1)
    assert stale in orc.weights(hub)[0] and not orc.live(stale) and named not in orc.weights(hub)[0]
    orc.close()


@needs_ref
@pytest.mark.parametrize("scene", GRAPH, ids=lambda s: s.name)
def test_oracle_equals_reference_graph(scene):
    if scene.refused:   # the reference has no bound: it runs the refused batch, and the one after it
        scene = copy.copy(scene)
        scene.steps = scene.steps + [("update", scene.refused), ("update", scene.after)]
    TC.run(scene, full=False, keys=scene.keys)


def _obs_play(scene):
    ref, model, slot_of = OO.RefObservations(), OS.ObsModel(scene, scene.keys), scene.slots()
    ref.set_kf_order(L.KM.rank(scene.keys[:scene.nkf]))
    try:
        lens = []
        for t, step in enumerate(scene.steps):
            model.apply(step)
            TO.ref_step(ref, model, step)
            if step[0] not in ("kf", "update"):
                ptr, _, _ = TO.compare(ref, model, scene, slot_of, list(range(len(model.obs))), (scene.name, t, step[0]), scene.keys)
                lens.append(np.diff(ptr))
                if step[0] == "pts":
                    row, last = model.kf_mp[0].copy(), {m: o.get(0) for m, o in enumerate(model.obs)}
        return model, lens, row, last
    finally:
        ref.close()


@needs_ref
@pytest.mark.parametrize("scene", L.obs_scenes(), ids=lambda s: s.name)
def test_observation_scenes(scene):
    """full row, cells of one point with the largest index observed, lists past 1024; oracle == reference"""
    model, lens, row, last = _obs_play(scene)
    cap = scene.facts["cap"]
    assert model.nfeat[0] == cap and (row >= 0).all()
    cells = {}
    for i, m in enumerate(row.tolist()):
        cells.setdefault(m, []).append(i)
    dup = [m for m, c in cells.items() if len(c) > 1]
    assert len(dup) == scene.facts["dup_cells"] and all(max(cells[m]) == last[m] for m in dup)
    assert lens[0][0] == scene.facts["long_len"][0] > 1024 and lens[0][1] == scene.facts["long_len"][1] > 1024
    assert lens[1][0] == lens[0][0] - 1    # keyframe 10 erased
    assert L._pow2ge(2 * cap) in (8192, 16384) and (cap != 4097 or L._pow2ge(2 * cap) >= 4 * cap - 4)


@needs_cull
def test_cull_scene():
    """2048 candidates; erases, kept candidates and points made bad along the list; oracle == reference"""
    scene = L.scene_cull()
    trace = []
    model = TK.run(scene, check_every=False, keys=scene.keys, trace=trace)
    (o,) = trace
    v = np.array(o["verdict"])
    assert len(v) == scene.facts["candidates"] == 2048
    assert model.nfeat[scene.facts["current"]] == scene.cap == 8192
    ne, nk = int((v == KC.ERASED).sum()), int((v == KC.KEPT).sum())
    assert ne >= 100 and nk >= 100, (ne, nk)
    assert len(o["bad_points"]) > 0
    first_e = int(np.flatnonzero(v == KC.ERASED)[0])
    assert (v[first_e + 1:] == KC.KEPT).any() and (v[:len(v) // 2] == KC.ERASED).any()


@needs_lm
@pytest.mark.parametrize("scene", L.lm_scenes(), ids=lambda s: s.name)
def test_local_map_scenes(scene):
    """n0 > 1024 counted keyframes; the maximum tied between slots in different tiles of 1024; oracle == reference"""
    trace = []
    got = TL.run(scene, check_every=False, keys=scene.keys, trace=trace)
    slot_of = scene.slots()
    f = scene.facts
    tied = f["tied"]
    assert len({int(slot_of[k]) // 1024 for k in tied}) >= 2
    want_ref = min(tied, key=lambda k: int(scene.keys[k]))
    for fm, lk, rk, lp in got:
        assert len(lk) == f["n0"] > 1024 and rk == want_ref
    assert want_ref != min(tied) and int(slot_of[want_ref]) // 1024 > min(int(slot_of[k]) for k in tied) // 1024
    if f["frame_cells"]:
        assert len(got) == 2 and len(got[1][0]) == f["frame_cells"]
