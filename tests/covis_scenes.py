"""Scripted maps for the covisibility graph (KeyFrame::UpdateConnections and SetBadFlag's connection half), shared by
tests/test_oracle_covis.py (oracle vs the reference's own KeyFrame.cc) and tests/test_gpu_covis.py (device vs oracle).

A scene is a list of steps on keyframes and map points named by creation index; the creation index is also the order key
(the reference's arena puts them in pointer order).  Each keyframe's slot is a seeded permutation of creation order, so
slot order is not key order.  `Model` replays the steps on plain arrays the way the reference changes its map
(MapPoint::AddObservation + KeyFrame::AddMapPoint, MapPoint::SetBadFlag, KeyFrame::EraseMapPointMatch, KeyFrame::SetBadFlag's
EraseObservation loop) and gives the inputs of orbfe_covis_update_connections_device.

Steps:
  ("kf", nfeatures)                  a new keyframe
  ("pts", ref_kfs, mp, kf, idx)      len(ref_kfs) new points, then the observations (mp[j], kf[j], idx[j]) in order
  ("update", [kf, ...])              UpdateConnections of each, in order (one device batch)
  ("erase_kf", kf)                   KeyFrame::SetBadFlag
  ("bad_pt", mp)                     MapPoint::SetBadFlag
  ("erase_match", kf, idx)           KeyFrame::EraseMapPointMatch(idx)"""
import numpy as np


class Scene:
    def __init__(self, name, cap, seed=0, max_connections=64):
        self.name, self.cap, self.steps, self.nkf, self.npts = name, int(cap), [], 0, 0
        self.seed, self.max_connections = seed, max_connections
        self.parent_set = set()   # keyframes whose first connection gave them a parent (only those may be erased)

    def kf(self, n=None):
        self.steps.append(("kf", self.cap if n is None else int(n)))
        self.nkf += 1
        return self.nkf - 1

    def pts(self, ref_kfs, obs):
        """new points with reference keyframes ref_kfs; obs = [(point offset into this call, kf, idx)]"""
        first = self.npts
        mp = np.array([first + o[0] for o in obs], np.int32)
        kf = np.array([o[1] for o in obs], np.int32)
        idx = np.array([o[2] for o in obs], np.int32)
        self.steps.append(("pts", np.asarray(ref_kfs, np.int32), mp, kf, idx))
        self.npts += len(ref_kfs)
        return first

    def update(self, kfs):
        self.steps.append(("update", [int(k) for k in kfs]))

    def erase_kf(self, kf):
        self.steps.append(("erase_kf", int(kf)))

    def bad_pt(self, mp):
        self.steps.append(("bad_pt", int(mp)))

    def erase_match(self, kf, idx):
        self.steps.append(("erase_match", int(kf), int(idx)))

    def slots(self):
        """slot of every keyframe: a seeded permutation of creation order"""
        return np.random.default_rng(1000 + self.seed).permutation(self.nkf).astype(np.int32)


class Model:
    """The scene's map as the reference holds it: mvpMapPoints per keyframe (point index, -1 = NULL), mObservations per
    point (dict kf -> feature; the reference's map iterates in key order), isBad per point.  keys[k] is keyframe k's order
    key (the creation index when None)."""

    def __init__(self, scene: Scene, keys=None):
        self.cap, self.keys = scene.cap, keys
        self.nfeat = []
        self._mp = np.zeros((0, scene.cap), np.int32)   # rows grow by doubling: kf_mp is its first len(nfeat) rows
        self.obs = []
        self.bad = np.zeros(0, bool)
        self.kf_bad = []
        self.mnid = []
        self.version = 0
        self._cache = None

    def apply(self, step, first_connected=lambda kf: True):
        op = step[0]
        self.version += 1
        if op == "kf":
            if len(self.nfeat) == len(self._mp):
                self._mp = np.vstack([self._mp, np.full((max(len(self._mp), 1), self.cap), -1, np.int32)])
            self.nfeat.append(step[1])
            self.kf_bad.append(False)
            self.mnid.append(len(self.mnid))
        elif op == "pts":
            _, ref, mp, kf, idx = step
            self.obs += [dict() for _ in range(len(ref))]
            self.bad = np.concatenate([self.bad, np.zeros(len(ref), bool)])
            for m, k, i in zip(mp.tolist(), kf.tolist(), idx.tolist()):
                self.obs[m][k] = i
                self.kf_mp[k, i] = m
        elif op == "bad_pt":
            self._point_bad(step[1])
        elif op == "erase_match":
            self.kf_mp[step[1], step[2]] = -1
        elif op == "erase_kf":
            kf = step[1]
            if self.mnid[kf] == 0:
                return
            for m in self.kf_mp[kf, :self.nfeat[kf]].tolist():
                if m < 0 or kf not in self.obs[m]:
                    continue
                del self.obs[m][kf]
                if len(self.obs[m]) <= 2:
                    self._point_bad(m)
            self.kf_bad[kf] = True
        else:
            self.version -= 1

    @property
    def kf_mp(self):
        return self._mp[:len(self.nfeat)]

    def key(self, k):
        """keyframe k's order key: mObservations, like every map keyed by KeyFrame*, iterates in this order"""
        return int(k) if self.keys is None else int(self.keys[k])

    def _point_bad(self, m):
        self.bad[m] = True
        for k, i in self.obs[m].items():
            self.kf_mp[k, i] = -1
        self.obs[m] = {}

    def inputs(self, slot_of, K):
        """(kf_mp [K*cap], counts [K], group_ptr, obs) in slot rows: the arrays orbfe_covis_update_connections_device takes"""
        if self._cache is not None and self._cache[0] == self.version:
            return self._cache[1]
        cap, n = self.cap, len(self.nfeat)
        kf_mp = np.full((K, cap), -1, np.int32)
        counts = np.zeros(K, np.int32)
        m = self.kf_mp.copy()
        if len(self.bad):
            mask = m >= 0
            m[mask & self.bad[np.where(mask, m, 0)]] = -1
        kf_mp[slot_of[:n]] = m
        counts[slot_of[:n]] = self.nfeat
        lens = np.array([len(o) for o in self.obs], np.int64)
        gp = np.zeros(len(self.obs) + 1, np.int32)
        gp[1:] = np.cumsum(lens)
        flat = np.zeros(int(gp[-1]), np.int32)
        pos = 0
        for o in self.obs:
            for k in sorted(o):
                flat[pos] = slot_of[k] * cap + o[k]
                pos += 1
        out = (kf_mp.ravel(), counts, gp, flat)
        self._cache = (self.version, out)
        return out


def _share(s, a, b, n, fa, fb, first_ref=None):
    """n new points seen by keyframes a (features fa..) and b (features fb..); returns the next free features"""
    s.pts([a] * n, [(j, a, fa + j) for j in range(n)] + [(j, b, fb + j) for j in range(n)])
    return fa + n, fb + n


def scene_initial_pair():
    s = Scene("initial_pair", 128, seed=1)
    a, b = s.kf(), s.kf()
    s.pts([a] * 100, [(j, a, j) for j in range(100)] + [(j, b, j) for j in range(100)])
    s.update([a, b])   # Tracking.cc:430-431: the root (mnId 0) gets no parent
    return s


def scene_local_mapping(seed=2, nkf=12, cap=160):
    """one update per new keyframe, each new keyframe sharing points with the last few; then a fuse-like edit"""
    rng = np.random.default_rng(seed)
    s = Scene("local_mapping", cap, seed=seed)
    free = []
    for k in range(nkf):
        s.kf()
        free.append(0)
        obs, ref = [], []
        for back in range(1, min(k, 4) + 1):
            n = int(rng.integers(3, 25))
            n = min(n, cap - free[k], cap - free[k - back])
            for j in range(n):
                obs += [(len(ref), k - back, free[k - back]), (len(ref), k, free[k])]
                if back > 1 and rng.random() < 0.5 and free[k - 1] < cap:   # some points seen by three keyframes
                    obs.append((len(ref), k - 1, free[k - 1]))
                    free[k - 1] += 1
                ref.append(k - back)
                free[k - back] += 1
                free[k] += 1
        if ref:
            s.pts(ref, obs)
        if k >= 1:
            s.update([k])
    # fuse-like edit: a match erased in the newest keyframe, a point made bad, points added between two old keyframes
    s.erase_match(nkf - 1, 0)
    s.bad_pt(1)
    if free[nkf - 3] + 20 <= cap and free[nkf - 1] + 20 <= cap:
        _share(s, nkf - 3, nkf - 1, 20, free[nkf - 3], free[nkf - 1])
    s.update([nkf - 1])
    return s


def scene_threshold():
    """shared counts of 14, 15 and 16, then all counts below 15 with a tied maximum"""
    s = Scene("threshold", 128, seed=3)
    k = [s.kf() for _ in range(5)]
    f = [0] * 5
    for other, n in ((1, 14), (2, 15), (3, 16)):
        f[4], f[other] = _share(s, 4, other, n, f[4], f[other])
    s.update([k[4]])
    s.update([k[1]])
    s.update([k[2]])
    return s


def scene_tied_max():
    s = Scene("tied_max", 64, seed=4)
    k = [s.kf() for _ in range(5)]
    f = [0] * 5
    for other, n in ((0, 7), (1, 9), (2, 9), (3, 3)):   # the maximum 9 twice: the smaller key wins
        f[4], f[other] = _share(s, 4, other, n, f[4], f[other])
    s.update([k[4]])
    s.update([k[3]])
    s.update([k[1], k[2]])
    return s


def scene_weight_ties():
    s = Scene("weight_ties", 128, seed=5)
    k = [s.kf() for _ in range(6)]
    f = [0] * 6
    for other in (0, 1, 2, 3, 4):
        f[5], f[other] = _share(s, 5, other, 20 if other != 2 else 17, f[5], f[other])
    s.update([k[5]])
    s.update([k[0], k[1], k[3]])
    return s


def scene_changed_unchanged():
    """A's own update keeps the filtered list; B sends A an unchanged weight (the list stays filtered); C sends A a changed
    weight (the list becomes the full sort, sub-threshold weights included)"""
    s = Scene("changed_unchanged", 128, seed=6)
    A, B, Cc, D = s.kf(), s.kf(), s.kf(), s.kf()
    f = [0] * 4
    f[A], f[B] = _share(s, A, B, 16, f[A], f[B])
    f[A], f[D] = _share(s, A, D, 5, f[A], f[D])
    f[A], f[Cc] = _share(s, A, Cc, 18, f[A], f[Cc])
    s.update([A])            # A: weights {B:16, C:18, D:5}, list [C, B]
    s.update([B])            # B -> A with 16: unchanged, A keeps its filtered list
    f[A], f[Cc] = _share(s, A, Cc, 2, f[A], f[Cc])
    s.update([Cc])           # C -> A with 20: changed, A's list is the full sort [C, B, D]
    s.update([D])            # D's only neighbour is A with 5 < 15: the maximum alone, A gets an unchanged 5
    return s


def scene_empty_and_duplicates():
    """an empty-counter call (no points; points only it sees), a point at two features of one keyframe, bad points"""
    s = Scene("empty_dup", 64, seed=7)
    a, b, c, d = s.kf(), s.kf(), s.kf(), s.kf()
    s.update([d])                                       # nothing at all
    s.pts([c] * 3, [(j, c, j) for j in range(3)])      # points only c sees
    s.update([c])
    first = s.pts([a] * 20, [(j, a, j) for j in range(20)] + [(j, b, j) for j in range(20)])
    s.pts([a], [(0, a, 30), (0, b, 30), (0, b, 31)])   # b holds the point at features 30 and 31
    s.pts([a] * 3, [(j, a, 40 + j) for j in range(3)] + [(j, c, 10 + j) for j in range(3)])
    s.update([a, b, d])
    s.bad_pt(first)
    s.bad_pt(first + 1)
    s.update([b, a])
    return s


def scene_batch30(seed=8):
    """30 keyframes that all see each other, updated in one batch in a shuffled order: every member is a neighbour of
    members before and after it"""
    rng = np.random.default_rng(seed)
    s = Scene("batch30", 256, seed=seed)
    n = 30
    ks = [s.kf() for _ in range(n)]
    free = [0] * n
    ref, obs = [], []
    for p in range(500):
        seen = rng.choice(n, size=int(rng.integers(2, 6)), replace=False)
        for k in seen:
            if free[k] < 256:
                obs.append((len(ref), int(k), free[k]))
                free[k] += 1
        ref.append(int(seen[0]))
    s.pts(ref, obs)
    order = rng.permutation(n).tolist()
    s.update(order)
    s.update(order[:7])
    return s


def scene_culling():
    """A names B asymmetrically (B's map never received A); erasing B leaves A's entry stale"""
    s = Scene("culling", 128, seed=9)
    A, B, Cc, E = s.kf(), s.kf(), s.kf(), s.kf()
    f = [0] * 4
    f[B], f[Cc] = _share(s, B, Cc, 20, f[B], f[Cc])
    f[A], f[E] = _share(s, A, E, 20, f[A], f[E])
    s.update([B])              # B: {C:20}, parent C
    f[A], f[B] = _share(s, A, B, 5, f[A], f[B])
    f[A], f[Cc] = _share(s, A, Cc, 25, f[A], f[Cc])
    s.update([A])              # A (mnId 0): {B:5, C:25, E:20}; B < 15 and not the maximum, so B's map does not name A
    f[A], f[E] = _share(s, A, E, 2, f[A], f[E])
    s.update([E])              # E -> A with 22, a changed weight: A's list is the full sort [C, E, B]
    s.erase_kf(B)              # EraseConnection on C only; A keeps B
    s.update([Cc])
    s.erase_kf(A)              # mnId 0: nothing
    return s


def scene_three_events():
    """a hub updated first in a batch, then three keyframes that each share 15 or more points with it: the hub's counter
    holds 3 entries and its map receives 3 events in the batch, the last from the newest keyframe (sorted with one padding
    entry, whatever the newest keyframe's key)"""
    s = Scene("three_events", 64, seed=14)
    hub, a, b, c = s.kf(), s.kf(), s.kf(), s.kf()
    f = [0] * 4
    for other, n in ((a, 15), (b, 17), (c, 16)):
        f[hub], f[other] = _share(s, hub, other, n, f[hub], f[other])
    s.update([hub, a, b, c])
    return s


def small_scenes():
    return [scene_initial_pair(), scene_local_mapping(), scene_threshold(), scene_tied_max(), scene_weight_ties(),
            scene_changed_unchanged(), scene_empty_and_duplicates(), scene_batch30(), scene_culling(), scene_three_events()]


def scene_large(nkf=2000, nfeat=2000, obs_per_point=8, window=12, batch=64, seed=11):
    """nkf keyframes x nfeat features, points seen by ~obs_per_point keyframes within +-window of a centre; every keyframe
    updated once, in batches of `batch` in creation order"""
    rng = np.random.default_rng(seed)
    s = Scene("large", nfeat, seed=seed)
    for _ in range(nkf):
        s.kf()
    npts = int(nkf * nfeat * 0.9) // obs_per_point
    centre = (np.arange(npts) * nkf) // npts
    offs = np.stack([rng.permutation(2 * window + 1)[:obs_per_point] for _ in range(npts)]) - window
    kfs = np.clip(centre[:, None] + offs, 0, nkf - 1)
    mp_l, kf_l, idx_l = [], [], []
    free = np.zeros(nkf, np.int64)
    for p in range(npts):
        for k in np.unique(kfs[p]).tolist():
            if free[k] < nfeat:
                mp_l.append(p)
                kf_l.append(k)
                idx_l.append(int(free[k]))
                free[k] += 1
    s.steps.append(("pts", centre.astype(np.int32), np.array(mp_l, np.int32), np.array(kf_l, np.int32), np.array(idx_l, np.int32)))
    s.npts = npts
    for b in range(0, nkf, batch):
        s.update(range(b, min(nkf, b + batch)))
    return s


def scene_capacity(max_connections=6):
    """one keyframe that sees exactly max_connections others, then one that sees max_connections + 1"""
    s = Scene("capacity", 64, seed=12, max_connections=max_connections)
    hub, hub2 = s.kf(), s.kf()
    f = {hub: 0, hub2: 0}
    others = [s.kf() for _ in range(max_connections + 1)]
    for o in others:
        f[o] = 0
    for o in others[:max_connections]:
        f[hub], f[o] = _share(s, hub, o, 3, f[hub], f[o])
    for o in others:
        f[hub2], f[o] = _share(s, hub2, o, 2, f[hub2], f[o])
    return s, hub, hub2
