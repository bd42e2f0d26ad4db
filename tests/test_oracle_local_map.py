"""CPU test of the UpdateReference oracle (oracle/orb_oracle_local_map.c): after every step of every scene of
tests/local_map_scenes.py, and for frames of 300, 1000 and 2000 matched points on the 2000 x 2000 map, the reference's own
Tracking::UpdateReference (oracle/_ref/libref_local_map.so) and the oracle, run on the same map with the reference's
ordered lists, agree on the frame's cells, mvpLocalKeyFrames, mpReferenceKF and mvpLocalMapPoints.  Also: each scene reaches
the case it is built for, and the oracle's statuses."""
import numpy as np
import pytest

import covis_scenes as S
import local_map_scenes as LS
from oracle import local_map as LM
from test_oracle_observations import ref_step as obs_ref_step

needs_ref = pytest.mark.skipif(not LM.ref_available(), reason="oracle/_ref/libref_local_map.so not built (needs the reference sources)")


def lm_inputs(model, slot_of, K):
    """the oracle's (and the device's) per-slot arrays from the model: the rows as the keyframes hold them, counts, live,
    keys (creation index) and point flags"""
    cap, n = model.cap, len(model.nfeat)
    kf_mp = np.full((K, cap), -1, np.int32)
    counts = np.zeros(K, np.int32)
    kf_mp[slot_of[:n]] = model.kf_mp
    counts[slot_of[:n]] = model.nfeat
    live, keys = np.zeros(K, np.uint8), np.zeros(K, np.uint64)
    live[slot_of[:n]] = model.live()
    keys[slot_of[:n]] = np.arange(n, dtype=np.uint64)
    return dict(kf_mp=kf_mp.ravel(), counts=counts, live=live, keys=keys, point_bad=model.bad.astype(np.uint8))


def oracle_local_map(a, cells, lists, K, cap):
    nb, nnb = LM.neighbours(lists, K)
    return LM.local_map(cells, a["point_bad"], a["kf_mp"], a["counts"], cap, a["live"], a["keys"], nb, nnb)


class RefRun:
    """a scene on the reference's own map and on the model"""

    def __init__(self, scene):
        self.scene, self.K, self.cap = scene, scene.nkf, scene.cap
        self.ref, self.model, self.slot_of = LM.RefLocalMap(), LS.LmModel(scene), scene.slots()

    def close(self):
        self.ref.close()

    def step(self, step):
        if step[0] == "to_be_erased":
            self.ref.to_be_erased(step[1])
        elif step[0] != "frame":
            self.model.apply(step)
            obs_ref_step(self.ref, self.model, step)

    def lists(self):
        """every keyframe's ordered list as the reference holds it, as slots"""
        so = self.slot_of
        return {int(so[k]): [int(so[v]) for v in self.ref.ordered(k)[0]] for k in range(len(self.model.nfeat))}

    def compare(self, cells, where):
        """the reference and the oracle on one frame; returns the reference's (cells, local keyframes, reference keyframe,
        local points) by creation index"""
        so = self.slot_of
        o = oracle_local_map(lm_inputs(self.model, so, self.K), cells, self.lists(), self.K, self.cap)
        fm, lk, rk, lp, _ = self.ref.update_reference(cells)
        assert o["status"] == 0, where
        assert o["frame_mp"].tolist() == fm.tolist(), (where, "frame cells")
        assert o["local_kf"].tolist() == [int(so[k]) for k in lk], (where, "local keyframes", lk)
        assert o["ref_kf"] == (int(so[rk]) if rk >= 0 else -1), (where, "reference keyframe", rk)
        assert o["local_points"].tolist() == lp, (where, "local points")
        return fm.tolist(), lk, rk, lp


def run(scene, check_every=True):
    r = RefRun(scene)
    got = []
    try:
        for t, step in enumerate(scene.steps):
            where = (scene.name, t, step[0])
            r.step(step)
            if step[0] == "frame":
                got.append(r.compare(step[1], where))
            elif check_every:
                r.compare(LS.probe_frame(r.model), where + ("probe",))
        return got
    finally:
        r.close()


@needs_ref
@pytest.mark.parametrize("scene", LS.small_scenes(), ids=lambda s: s.name)
def test_oracle_equals_reference_local_map(scene):
    run(scene)


@needs_ref
def test_scenes_reach_their_cases():
    """each scene's frames give the lists its docstring names (so it fails under the wrong variant it is built against)"""
    got = {s.name: run(s, check_every=False) for s in LS.small_scenes()}
    # tie and double vote: keyframes 0 (K0), 1 (x), 2 (y)
    tie = got["tie_double_vote"]
    assert [f[2] for f in tie] == [0, 0, 1, 1] and tie[0][1] == [0, 1, 2] and tie[2][1] == [0, 1, 2] and tie[3][1] == [1, 2, 0]
    # the empty counter: NULL cells only, a bad point only, a point whose only observer is retired
    eb = got["empty_bad"]
    assert all(f[1] == [] and f[2] == -1 and f[3] == [] for i, f in enumerate(eb) if i in (0, 1, 2, 4))
    assert eb[2][0] == [-1] and eb[3][0][0] == -1 and eb[3][0][3] == -1 and eb[3][1] == [1, 2, 3]
    # the bound: n0 = 79 and 80 end at 81 entries, 81 and 100 append nothing
    for n0, want in ((79, 81), (80, 81), (81, 81), (100, 100)):
        for f in got["bound%d" % n0]:
            assert len(f[1]) == want and f[1][:n0] == list(range(1, n0 + 1)), n0
    assert got["bound79"][0][1][79:] == [80, 81] and got["bound80"][0][1][80:] == [81]
    # listed entries: c1 = 1, c2 = 2, b = 3, d = 4, e = 5, hub = 6, its neighbours 7 .. 17
    ll = got["listed_limits"]
    assert ll[0][1] == [1, 2, 3, 4]
    assert ll[1][1] == [6] + list(range(7, 17))              # the 11th neighbour (17) is not among the first 10
    assert ll[2][1] == [6] + list(range(7, 16)) + [16]       # the 10th (16) is appended for the hub
    # stale: c = 1, r = 2, h2 = 4, t = 6
    st = got["stale"]
    assert st[0][1] == [1, 2] and st[1][1] == [1, 4] and st[2][1] == [1, 6, 4] and st[3][1] == [1, 6, 4]
    # rows: a point named twice in a row is listed once, a queued keyframe's row is not read until it is processed
    rw = got["rows"]
    assert all(len(f[3]) == len(set(f[3])) for f in rw) and 3 not in rw[0][1] and 3 in rw[2][1]


@needs_ref
def test_oracle_equals_reference_large_map():
    """2000 keyframes x 2000 features: frames of 300, 1000 and 2000 matched points around keyframe 1000"""
    scene = S.scene_large()
    r = RefRun(LS.LmScene("large", scene.cap, seed=scene.seed))
    r.scene, r.K, r.slot_of = scene, scene.nkf, scene.slots()
    r.model = LS.LmModel(scene)
    try:
        for step in scene.steps:
            r.step(step)
        for cells in LS.large_frames(r.model, r.slot_of):
            fm, lk, rk, lp = r.compare(cells, ("large", len(cells)))
            assert len(lk) > 10 and len(lp) > len(set(cells.tolist()))
    finally:
        r.close()


def test_oracle_statuses():
    """a frame cell or a live row's value >= npoints, or a live slot's count outside 0 .. cap: -1; a retired slot's row is
    not read"""
    cap, K = 4, 3
    kf_mp = np.array([0, 1, 2, -1, 0, 1, -1, -1, 2, 2, -1, -1], np.int32)
    counts = np.array([3, 2, 2], np.int32)
    live, keys = np.ones(K, np.uint8), np.array([2, 0, 1], np.uint64)
    pb = np.zeros(3, np.uint8)
    nb, nnb = LM.neighbours({}, K)

    def call(cells=(0, 2), **kw):
        a = dict(point_bad=pb, kf_mp=kf_mp, counts=counts, cap=cap, live=live, keys=keys, nb=nb, nnb=nnb)
        a.update(kw)
        return LM.local_map(np.array(cells, np.int32), **a)

    ok = call()
    assert ok["status"] == 0 and ok["local_kf"].tolist() == [1, 2, 0] and ok["ref_kf"] == 0
    assert ok["local_points"].tolist() == [0, 1, 2]
    assert call(cells=(0, 3))["status"] == -1
    assert call(kf_mp=np.where(kf_mp == 2, 3, kf_mp))["status"] == -1
    assert call(counts=np.array([3, 5, 2], np.int32))["status"] == -1
    assert call(counts=np.array([3, 5, 2], np.int32), live=np.array([1, 0, 1], np.uint8))["status"] == 0
