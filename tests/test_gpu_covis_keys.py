"""GPU tests of the covisibility graph and its readers (orbfe_covis_*) on pointer-sized order keys
(tests/covis_key_scenes.py): the tests of test_gpu_covis.py, test_gpu_observations.py, test_gpu_kf_culling.py and
test_gpu_local_map.py, run on their own Run classes with keys that use the high word, straddle the low word's wrap and 2^63,
reach 2^64 - 1 and order keyframes against creation and slot order.  The oracle they are compared with is pinned to the
reference under the same keys by tests/test_oracle_covis_keys.py.  Also: a key equal to that of a retired slot a weight map
still names is refused with nothing changed, and accepted once no map names it; keys 0 and 2^64 - 1 in one add."""
import numpy as np
import pytest

import orb_slam_b200 as fe
from orb_slam_b200 import bow as B

import covis_key_scenes as KM
import covis_scenes as S
import kf_culling_scenes as KS
import local_map_scenes as LS
import observation_scenes as OS
import test_gpu_covis as GC
import test_gpu_kf_culling as GK
import test_gpu_local_map as GL
import test_gpu_observations as GO

pytestmark = pytest.mark.gpu
MAPS = [m for m in KM.NAMES if m != "small"]


def _covis(scene, keys):
    r = GC.Run(scene, keys=keys)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            r.check((scene.name, t, step[0]))
    finally:
        r.close()


def _observations(scene, keys):
    r = GO.Run(scene, keys)
    rng = np.random.default_rng(7)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            r.check((scene.name, t, step[0]), rng)
    finally:
        r.close()


FAMILIES = {
    "covis": (S.small_scenes, _covis),
    "observations": (OS.small_scenes, _observations),
    "kf_culling": (KS.small_scenes, lambda sc, keys: GK._play(sc, keys=keys).close()),
    "local_map": (LS.small_scenes, lambda sc, keys: GL._play(sc, keys=keys).close()),
}


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", MAPS)
def test_device_equals_oracle_under_every_key_map(gpu_required, family, name):
    """every small scene of the family, the device equal to the oracle after every step"""
    scenes, play = FAMILIES[family]
    for scene in scenes():
        play(scene, KM.keys(name, scene.nkf))


def test_large_map_under_wrap32(gpu_required):
    """2000 keyframes x 2000 features, the low word wrapping at keyframe 1000: covis batches of 64, every point's
    observations, one cull and one local map"""
    scene = S.scene_large()
    keys = KM.keys("wrap32", scene.nkf)
    r = GC.Run(scene, max_batch=64, keys=keys)
    try:
        for t, step in enumerate(scene.steps):
            r.step(step)
            if step[0] == "update":
                r.check(("large", t))
    finally:
        r.close()
    o = GO.Run(scene, keys)
    try:
        for step in scene.steps:
            o.step(step)
        o.check("large", np.random.default_rng(8))
    finally:
        o.close()
    GK._play(KS.large_culls(S.scene_large(), currents=(1000,)), check_all=False, keys=keys).close()
    m = GL._play(scene, check_all=False, keys=keys)
    try:
        cells = next(iter(LS.large_frames(m.model, m.slot_of, sizes=(1000,))))
        out, _ = m.check(cells, ("large", len(cells)))
        assert len(out["local_kf"]) > 10
    finally:
        m.close()


@pytest.mark.parametrize("name", ["top", "interleaved"])
def test_batch_equals_batches_of_one(gpu_required, name):
    scene = S.scene_batch30()
    keys = KM.keys(name, scene.nkf)
    a, b = GC.Run(scene, max_batch=64, keys=keys), GC.Run(scene, single=True, max_batch=64, keys=keys)
    try:
        for step in scene.steps:
            a.step(step)
            b.step(step)
        assert GC.state(a.g, a.K) == GC.state(b.g, b.K) == GC.oracle_state(a.orc, a.K)
    finally:
        a.close()
        b.close()


def test_stale_key_is_refused_until_no_map_names_it(gpu_required):
    """scene_culling leaves A's map naming the retired B.  A new keyframe in a free slot with B's key is refused
    (ORBFE_ERR_ARG, reported once, the graph unchanged); after A's own update drops B the same add succeeds, and the graph
    equals the oracle's"""
    scene = S.scene_culling()
    scene.nkf += 1                   # one slot that no step adds: the new keyframe's
    keys = KM.keys("random", scene.nkf)
    r = GC.Run(scene, keys=keys)
    try:
        for step in scene.steps:
            r.step(step)
        A, Bk, new = 0, 1, scene.nkf - 1
        sa, sn = int(r.slot_of[A]), int(r.slot_of[new])
        assert -1 in GC.export(r.g, [sa], 1, 0)[1].tolist()   # A's map names the retired B
        before = GC._snapshot(r)
        with pytest.raises(fe.OrbfeError) as e:
            r.g.add([sn], [new], [int(keys[Bk])])
        assert e.value.code == fe.ORBFE_ERR_ARG
        r.g.sync()                   # reported once: nothing pending
        assert GC._snapshot(r) == before
        r.g.add([sn], [new], [int(keys[new])])   # another key is accepted in the same slot ...
        r.g.erase(sn)                # ... and retired again, named by no map
        r.step(("update", [A]))      # A's own update: B is no longer among its observers
        assert GC._snapshot(r) == GC.oracle_state(r.orc, r.K)
        r.g.add([sn], [new], [int(keys[Bk])])
        r.orc.add(sn, new, int(keys[Bk]))
        r.check("after the stale entry is gone")
    finally:
        r.close()


def test_keys_zero_and_max_in_one_add(gpu_required):
    """keys 0 and 2^64 - 1 in one add are accepted; on scene_three_events with the maximal key first, the 3-entry counter
    and the 3 events of the hub (each sorted with one padding entry) equal the oracle"""
    g = B.CovisibilityGraph(4, 8, 4)
    try:
        g.add([2, 0], [0, 1], [0, KM.MAX])
        g.sync()
    finally:
        g.close()
    scene = S.scene_three_events()
    for keys in ([KM.MAX, 0, 1 << 63, 5], [5, 0, 1 << 63, KM.MAX], [0, 1 << 63, KM.MAX, 5]):
        _covis(scene, np.array(keys, np.uint64))
