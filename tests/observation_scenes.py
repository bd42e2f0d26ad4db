"""Scripted maps for MapPoint::GetObservations() built from the keyframes' rows (orbfe_covis_observations_device), shared by
tests/test_oracle_observations.py (oracle vs the reference's own MapPoint.cc / KeyFrame.cc) and tests/test_gpu_observations.py
(device vs oracle).  Reuses tests/covis_scenes.py: the scenes are covis_scenes.Scene step lists with the steps below added,
and ObsModel is covis_scenes.Model with mpRefKF and the observer set kept as well.

A keyframe becomes an observer when its observations are added: a ("kf", n) keyframe at once (Tracking's initial pair and
the scripted maps of covis_scenes), a ("kfq", n) keyframe only at its ("process", kf) step.  New steps:
  ("kfq", nfeatures)        a keyframe in LocalMapping's queue: a row, no observations, not an observer
  ("row", kf, idx, mp)      KeyFrame::AddMapPoint(mp, idx) alone (Tracking fills a new keyframe's matches)
  ("process", kf)           ProcessNewKeyFrame: AddObservation(kf, i) for every i ascending whose point is not bad
  ("observe", mp, kf, idx)  AddObservation + AddMapPoint of an existing point (Fuse's add branch)
  ("replace", a, b)         MapPoint::Replace: a's observations move to b, or a's cell is erased where b is already there
  ("ba_erase", kf, mp)      the local-BA outlier pair EraseMapPointMatch(mp) + EraseObservation(kf); mpRefKF moves to the
                            first remaining observer when it was kf
A ("row", ...) on a cell whose point still lists the keyframe is the one edit no reference path makes: the row then stops
naming the old point while the old point's mObservations keeps the keyframe (see DESIGN.md §2).  covis_scenes'
("erase_match", ...) alone does the same to the erased point; ObsModel.divergent collects the points these two edits touch."""
import numpy as np

import covis_scenes as S


class ObsScene(S.Scene):
    def kfq(self, n=None):
        self.steps.append(("kfq", self.cap if n is None else int(n)))
        self.nkf += 1
        return self.nkf - 1

    def row(self, kf, idx, mp):
        self.steps.append(("row", int(kf), int(idx), int(mp)))

    def process(self, kf):
        self.steps.append(("process", int(kf)))

    def observe(self, mp, kf, idx):
        self.steps.append(("observe", int(mp), int(kf), int(idx)))

    def replace(self, a, b):
        self.steps.append(("replace", int(a), int(b)))

    def ba_erase(self, kf, mp):
        self.steps.append(("ba_erase", int(kf), int(mp)))


class ObsModel(S.Model):
    """Model plus mpRefKF per point (-2 where the reference's pointer is undefined) and the observer flag per keyframe."""

    def __init__(self, scene, keys=None):
        super().__init__(scene, keys)
        self.ref = []
        self.observer = []
        self.divergent = set()   # the old and new point of a row overwrite: mObservations and the rows disagree on them

    def apply(self, step, first_connected=lambda kf: True):
        op = step[0]
        if op in ("kf", "kfq"):
            super().apply(("kf", step[1]))
            self.observer.append(op == "kf")
            return
        if op == "pts":
            self.ref += step[1].tolist()
            super().apply(step)
            return
        if op == "erase_kf":
            self.version += 1
            self._erase_kf(step[1])
            return
        if op == "erase_match":   # EraseMapPointMatch(idx) alone (covis_scenes' fuse-like edit) leaves mObservations as it is
            old = int(self.kf_mp[step[1], step[2]])
            if old >= 0 and self.obs[old].get(step[1]) == step[2]:
                self.divergent.add(old)
        if op not in ("row", "process", "observe", "replace", "ba_erase"):
            super().apply(step)
            return
        self.version += 1
        if op == "row":
            _, kf, idx, mp = step
            old = int(self.kf_mp[kf, idx])
            if old >= 0 and old != mp and kf in self.obs[old] and self.obs[old][kf] == idx:
                self.divergent.update((old, mp))
            self.kf_mp[kf, idx] = mp
        elif op == "process":
            kf = step[1]
            for i in range(self.nfeat[kf]):
                m = int(self.kf_mp[kf, i])
                if m >= 0 and not self.bad[m]:
                    self.obs[m][kf] = i
            self.observer[kf] = True
        elif op == "observe":
            _, m, kf, idx = step
            self.obs[m][kf] = idx
            self.kf_mp[kf, idx] = m
        elif op == "replace":
            a, b = step[1], step[2]
            if a == b:
                return
            moved, self.obs[a] = self.obs[a], {}
            self.bad[a] = True
            for k in sorted(moved):
                i = moved[k]
                if k in self.obs[b]:
                    self.kf_mp[k, i] = -1
                else:
                    self.kf_mp[k, i] = b
                    self.obs[b][k] = i
        elif op == "ba_erase":
            kf, m = step[1], step[2]
            if kf in self.obs[m]:
                self.kf_mp[kf, self.obs[m][kf]] = -1
            self._erase_observation(m, kf)

    def _erase_observation(self, m, kf):
        """MapPoint::EraseObservation"""
        if kf not in self.obs[m]:
            return
        del self.obs[m][kf]
        if self.ref[m] == kf:
            self.ref[m] = min(self.obs[m], key=self.key) if self.obs[m] else -2   # mObservations.begin()->first
        if len(self.obs[m]) <= 2:
            self._point_bad(m)

    def _erase_kf(self, kf):
        """KeyFrame::SetBadFlag's EraseObservation loop (mnId 0 returns at once)"""
        if self.mnid[kf] == 0:
            return
        for m in self.kf_mp[kf, :self.nfeat[kf]].tolist():
            if m >= 0:
                self._erase_observation(m, kf)
        self.kf_bad[kf] = True

    def live(self):
        """keyframes that are observers and not bad"""
        return np.array([o and not b for o, b in zip(self.observer, self.kf_bad)], bool)


def _pair(s, a, b, n, fa, fb, extra=()):
    """n new points seen by a (features fa..) and b (fb..) and by every (kf, first feature) of extra; reference keyframe a"""
    obs = [(j, a, fa + j) for j in range(n)] + [(j, b, fb + j) for j in range(n)]
    for k, f in extra:
        obs += [(j, k, f + j) for j in range(n)]
    return s.pts([a] * n, obs)


def scene_process_new_keyframe():
    """the initial pair, then keyframes that wait in the queue with rows filled (one names a point at two features, one a
    point that becomes bad before processing) and become observers at ProcessNewKeyFrame"""
    s = ObsScene("process_new_keyframe", 64, seed=21)
    a, b = s.kf(), s.kf()
    first = _pair(s, a, b, 30, 0, 0)
    s.update([a, b])
    c = s.kfq()
    for j in range(12):
        s.row(c, j, first + j)
    s.row(c, 40, first + 3)            # first + 3 at features 3 and 40 of c: the larger index is the observation
    s.row(c, 41, first + 20)
    s.row(c, 20, first + 20)           # and first + 20 at 41 and 20: the larger index comes first in the row
    s.row(c, 30, first + 25)
    s.bad_pt(first + 25)               # culled while c waits: ProcessNewKeyFrame skips it
    d = s.kfq()                        # queued behind c
    for j in range(6):
        s.row(d, j, first + j)
    s.process(c)
    s.update([c])
    s.process(d)
    s.update([d])
    return s


def scene_fuse():
    """Fuse: the add branch, Replace in both directions (the point with fewer observations is replaced), the erase branch
    where the target already sees a keyframe, and chains of replaces"""
    s = ObsScene("fuse", 64, seed=22)
    k = [s.kf() for _ in range(5)]
    f = [0] * 5
    p = _pair(s, k[0], k[1], 6, f[0], f[1], extra=[(k[2], f[2])])    # p..p+5: seen by 0, 1, 2
    f = [6, 6, 6, 0, 0]
    q = _pair(s, k[3], k[4], 6, f[3], f[4])                           # q..q+5: seen by 3, 4
    f[3] = f[4] = 6
    r = _pair(s, k[2], k[3], 6, 10, 10, extra=[(k[4], 10)])           # r..r+5: seen by 2, 3, 4 (2 shared with p)
    s.update(k)
    s.observe(q, k[0], 20)             # fuse add: q gains keyframe 0
    s.replace(q + 1, p + 1)            # q+1 (3, 4) -> p+1 (0, 1, 2): no common keyframe, every cell moves
    s.replace(p + 2, r + 2)            # p+2 (0, 1, 2) -> r+2 (2, 3, 4): keyframe 2 is common, its cell is erased
    s.replace(q + 3, p + 3)            # chain: q+3 -> p+3 -> r+3
    s.replace(p + 3, r + 3)
    s.replace(r + 4, q + 4)            # the other direction: a point with more observations replaced by one with fewer
    s.replace(q + 4, q + 4)            # the same point: nothing
    s.update(k)
    return s


def scene_culling():
    """MapPointCulling (SetBadFlag of points) and KeyFrameCulling (SetBadFlag of keyframes): observations leave, points
    with two or fewer become bad, mpRefKF moves off an erased keyframe"""
    s = ObsScene("culling", 64, seed=23)
    k = [s.kf() for _ in range(5)]
    p = _pair(s, k[1], k[2], 10, 0, 0, extra=[(k[3], 0), (k[4], 0)])   # seen by 1..4, reference keyframe 1
    t = _pair(s, k[0], k[1], 10, 0, 10, extra=[(k[2], 10)])            # seen by 0, 1, 2
    s.update(k)
    s.bad_pt(p)
    s.bad_pt(t + 1)
    s.erase_kf(k[1])                   # p+1..: 3 observers left, reference moves to 2; t+..: 2 left, bad
    s.update([k[0], k[2], k[3], k[4]])
    s.erase_kf(k[3])                   # p+..: 2 observers left: bad
    return s


def scene_ba_outliers():
    """local-BA outliers: EraseMapPointMatch + EraseObservation of a non-reference observer, of the reference one (mpRefKF
    moves to the first remaining keyframe), and down to two observers (the point becomes bad)"""
    s = ObsScene("ba_outliers", 64, seed=24)
    k = [s.kf() for _ in range(6)]
    p = _pair(s, k[2], k[0], 8, 0, 0, extra=[(k[1], 0), (k[3], 0), (k[4], 0), (k[5], 0)])   # seen by 0..5, reference 2
    s.update(k)
    s.ba_erase(k[4], p)
    s.ba_erase(k[2], p + 1)            # the reference keyframe: mpRefKF -> keyframe 0
    s.ba_erase(k[0], p + 1)            # the new reference again: -> keyframe 1
    s.ba_erase(k[5], p + 2)
    s.ba_erase(k[3], p + 2)
    s.ba_erase(k[1], p + 2)            # 5 -> 2 observers: bad
    s.ba_erase(k[1], p + 3)            # not the reference, then the reference
    s.ba_erase(k[2], p + 3)
    s.update(k)
    return s


def scene_queued():
    """a queued keyframe's row names points for several steps (updates of others, a cull) before it is processed"""
    s = ObsScene("queued", 64, seed=25)
    a, b, c = s.kf(), s.kf(), s.kf()
    p = _pair(s, a, b, 20, 0, 0, extra=[(c, 0)])
    s.update([a, b, c])
    q1, q2 = s.kfq(), s.kfq()
    for j in range(20):
        s.row(q1, j, p + j)
        s.row(q2, 19 - j, p + j)
    s.update([a])
    s.bad_pt(p + 5)
    s.process(q2)
    s.update([q2])
    s.process(q1)
    s.update([q1])
    return s


def scene_overwritten_cell():
    """a row cell overwritten while its old point still lists the keyframe (no reference path does this): the rows stop
    naming the old point, the old point's mObservations keeps the keyframe"""
    s = ObsScene("overwritten_cell", 32, seed=26)
    a, b, c = s.kf(), s.kf(), s.kf()
    p = _pair(s, a, b, 4, 0, 0, extra=[(c, 0)])
    n = _pair(s, a, c, 2, 10, 10)
    s.row(b, 1, n)                     # b's feature 1 now names n; p+1 still lists b at 1
    return s


def small_scenes():
    return [scene_process_new_keyframe(), scene_fuse(), scene_culling(), scene_ba_outliers(), scene_queued(), scene_overwritten_cell()]


def covis_scenes_as_obs():
    """the scenes of covis_scenes (every keyframe an observer from its creation)"""
    return S.small_scenes()
