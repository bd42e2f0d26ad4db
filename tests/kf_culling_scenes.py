"""Scripted maps for LocalMapping::KeyFrameCulling with SetBadFlag's map-point half (orbfe_covis_keyframe_culling_device),
shared by tests/test_oracle_kf_culling.py (oracle vs the reference's own LocalMapping.cc) and tests/test_gpu_kf_culling.py
(device vs oracle).  The scenes are observation_scenes.ObsScene step lists with two steps added:
  ("octave", kf, idx, octaves)     GetKeyPointUn(idx[j]).octave = octaves[j] (every keypoint starts at octave 0)
  ("cull", current, not_erase)     KeyFrameCulling() with `current` as mpCurrentKeyFrame; the keyframes of not_erase carry
                                   mbNotErase
CullModel is ObsModel with the octaves kept; a cull step's model is ObsModel._erase_kf for the keyframes it erased, in list
order (CullModel.apply takes them: the verdicts come from the reference or the oracle).

Every scene starts with K0 (mnId 0) and the current keyframe c, and updates its keyframes after the points are made, c
last, so c's list holds every keyframe sharing at least 15 points with it (weight descending, the larger key first on a tie).
Keyframes that only help (observers) carry 40 points of their own seen by K0 alone besides, so they are never redundant."""
import numpy as np

import observation_scenes as OS


class CullScene(OS.ObsScene):
    def __init__(self, name, cap=128, seed=0, max_connections=64):
        super().__init__(name, cap, seed=seed, max_connections=max_connections)
        self.free = []

    def kf(self, n=None):
        self.free.append(0)
        return super().kf(n)

    def kfq(self, n=None):
        self.free.append(0)
        return super().kfq(n)

    def octave(self, kf, idx, octaves):
        self.steps.append(("octave", int(kf), np.asarray(idx, np.int32), np.asarray(octaves, np.int32)))

    def cull(self, current, not_erase=()):
        self.steps.append(("cull", int(current), tuple(int(k) for k in not_erase)))

    def seen(self, n, kfs, ref=None, octaves=None):
        """n new points, each seen by every keyframe of kfs at its next free features; reference keyframe ref (default
        kfs[0]); octaves = {kf: octave} for the new cells.  Returns the first point."""
        obs, cells = [], {}
        for k in kfs:
            cells[k] = list(range(self.free[k], self.free[k] + n))
            obs += [(j, k, self.free[k] + j) for j in range(n)]
            self.free[k] += n
            assert self.free[k] <= self.cap
        first = self.pts([kfs[0] if ref is None else ref] * n, obs)
        for k, o in (octaves or {}).items():
            self.octave(k, cells[k], [o] * n)
        return first

    def helpers(self, k0, hs, n=40):
        for h in hs:
            self.seen(n, [h, k0])


class CullModel(OS.ObsModel):
    """ObsModel plus every keyframe's octaves."""

    def __init__(self, scene):
        super().__init__(scene)
        self.oct = np.zeros((0, scene.cap), np.int32)

    def apply(self, step, erased=()):
        op = step[0]
        if op in ("kf", "kfq"):
            self.oct = np.vstack([self.oct, np.zeros((1, self.cap), np.int32)])
        if op == "octave":
            self.oct[step[1], step[2]] = step[3]
            return
        if op == "cull":
            self.version += 1
            for kf in erased:
                self._erase_kf(kf)
            return
        super().apply(step)


def _start(name, seed, cap=128):
    s = CullScene(name, cap, seed=seed)
    return s, s.kf(), s.kf()


def _finish(s, k0, c, rest):
    s.update([k0] + list(rest))
    s.update([c])


def scene_nothing_redundant():
    """no candidate reaches the ratio: points with three observers, and four with one of them too coarse"""
    s, k0, c = _start("nothing_redundant", 31)
    h1, h2, a, b = (s.kf() for _ in range(4))
    s.helpers(k0, [h1, h2])
    s.seen(20, [a, c, h1])
    s.seen(20, [b, c, h1, h2], octaves={h2: 2})
    _finish(s, k0, c, [h1, h2, a, b])
    s.cull(c)
    return s


def scene_ratio_boundary():
    """18 of 20 redundant is kept (18 > 18.0 is false), 20 of 20 is erased, and a keyframe whose points all went bad
    (0 of 0) is kept"""
    s, k0, c = _start("ratio_boundary", 32)
    h1, h2, a, b, z = (s.kf() for _ in range(5))
    s.helpers(k0, [h1, h2])
    s.seen(18, [a, c, h1, h2])
    s.seen(2, [a, c])
    s.seen(20, [b, c, h1, h2])
    zp = s.seen(16, [z, c])
    _finish(s, k0, c, [h1, h2, a, b, z])
    for j in range(16):
        s.bad_pt(zp + j)
    s.cull(c)
    return s


def scene_observations_3_4():
    """Observations() == 3 is not redundant, == 4 is"""
    s, k0, c = _start("observations_3_4", 33)
    h1, h2, a, b = (s.kf() for _ in range(4))
    s.helpers(k0, [h1, h2])
    s.seen(20, [a, c, h1])
    s.seen(20, [b, c, h1, h2])
    _finish(s, k0, c, [h1, h2, a, b])
    s.cull(c)
    return s


def scene_octave_gate():
    """the candidates' cells at octave 2; one observer at octave 3 (level+1: counts) or at 4 (level+2: does not)"""
    s, k0, c = _start("octave_gate", 34)
    h1, h2, a, b = (s.kf() for _ in range(4))
    s.helpers(k0, [h1, h2])
    s.seen(20, [a, c, h1, h2], octaves={a: 2, h2: 3})
    s.seen(20, [b, c, h1, h2], octaves={b: 2, h2: 4})
    _finish(s, k0, c, [h1, h2, a, b])
    s.cull(c)
    return s


def scene_duplicate_cells():
    """two points each at two cells of the candidate, octaves 0 and 2, their observers at 2: each counts twice, redundant
    only at its octave-2 cell, so 15 of 17 is kept (one count per point, 15 of 15, would erase it)"""
    s, k0, c = _start("duplicate_cells", 35)
    h1, h2, a = (s.kf() for _ in range(3))
    s.helpers(k0, [h1, h2])
    p = s.seen(2, [a, c, h1, h2], octaves={c: 2, h1: 2, h2: 2})   # a's cells at octave 0
    for j in range(2):
        s.observe(p + j, a, s.free[a])     # a names it again at a later feature: the observation's index
        s.octave(a, [s.free[a]], [2])
        s.free[a] += 1
    s.seen(13, [a, c, h1, h2])
    _finish(s, k0, c, [h1, h2, a])
    s.cull(c)
    return s


def scene_order():
    """b (first: the larger key on a tie) erased takes a's points to three observers: a is kept; e (first: the heavier)
    erased makes two of d's points bad: d's 16 of 16 is erased where 16 of 18 was not"""
    s, k0, c = _start("order", 36)
    h1, h2, a, b, d, e = (s.kf() for _ in range(6))
    s.helpers(k0, [h1, h2])
    s.seen(20, [a, b, c, h1])
    s.seen(20, [e, c, h1, h2])
    s.seen(2, [e, d, c])
    s.seen(16, [d, c, h1, h2])             # d: 16 of 18 is kept (16 > 16.2 is false); e weighs 22 with c, d 18
    _finish(s, k0, c, [h1, h2, a, b, d, e])
    s.cull(c)
    return s


def scene_id0_and_not_erase():
    """K0 (mnId 0) and a keyframe with mbNotErase are both redundant: skipped and kept with mbToBeErased"""
    s, k0, c = _start("id0_not_erase", 37)
    h1, h2, n = (s.kf() for _ in range(3))
    s.helpers(k0, [h1, h2])
    s.seen(20, [k0, c, h1, h2])
    s.seen(20, [n, c, h1, h2])
    _finish(s, k0, c, [h1, h2, n])
    s.cull(c, not_erase=[n])
    return s


def scene_stale():
    """two keyframes retired while c's list still names them (c's list is the full sort, their maps never named c):
    r2's points still have four observers (a repeat), r1's 9 of 10 with four and one with three (kept)"""
    s, k0, c = _start("stale", 38)
    h1, h2, x, r1, r2 = (s.kf() for _ in range(5))
    s.helpers(k0, [h1, h2])
    for r in (r1, r2):
        s.seen(3, [r, h1])
    s.update([k0, h1, h2, r1, r2])         # r's first connection: parent h1, its map {h1, ..} only
    s.seen(9, [r1, c, h1, h2, x])
    s.seen(1, [r1, c, h1, h2])
    s.seen(10, [r2, c, h1, h2, x])
    s.seen(20, [c, h1, h2])
    s.update([c])                          # r1, r2 weigh 10 < 15: c's list is filtered, their maps do not get c
    s.seen(16, [x, c])
    s.update([x])                          # x -> c with a new weight: c's list becomes the full sort, r1 and r2 included
    s.erase_kf(r1)
    s.erase_kf(r2)
    s.cull(c)
    return s


def scene_ref_and_cascade():
    """e is erased: mpRefKF moves off e to the smallest remaining key, a point seen by e alone loses its last observer
    (bad, mpRefKF left undefined), a point seen by e, c and l goes bad and both of l's cells naming it become NULL; a
    queued keyframe's row naming that point is left as it is"""
    s, k0, c = _start("ref_and_cascade", 39)
    h1, h2, l, e = (s.kf() for _ in range(4))
    s.helpers(k0, [h1, h2, l])
    s.seen(20, [h2, h1, e, c])             # keys h1 < h2 < e: created in that order; ref e below
    s.seen(10, [e, c, h1, h2], ref=e)
    s.seen(1, [e], ref=e)
    q = s.seen(1, [e, c, l], ref=e)
    s.observe(q, l, s.free[l])             # l names q twice, the observation at the later cell
    s.free[l] += 1
    s.seen(8, [e, c, h1, h2, l], ref=e)
    qk = s.kfq()
    s.row(qk, 0, q)
    _finish(s, k0, c, [h1, h2, l, e])
    s.cull(c)
    s.process(qk)
    return s


def small_scenes():
    return [scene_nothing_redundant(), scene_ratio_boundary(), scene_observations_3_4(), scene_octave_gate(), scene_duplicate_cells(),
            scene_order(), scene_id0_and_not_erase(), scene_stale(), scene_ref_and_cascade()]


def large_culls(scene, currents=(1000, 500)):
    """covis_scenes.scene_large (2000 keyframes x 2000 features) with culls for the current keyframes given"""
    for k in currents:
        scene.steps.append(("cull", int(k), ()))
    return scene
