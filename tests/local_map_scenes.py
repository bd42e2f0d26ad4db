"""Scripted maps for Tracking::UpdateReference (orbfe_covis_local_map_device), shared by tests/test_oracle_local_map.py (oracle
vs the reference's own Tracking.cc) and tests/test_gpu_local_map.py (device vs oracle).  The scenes are kf_culling_scenes'
CullScene step lists (keyframes and points by creation index, slots a seeded permutation of creation order, so slot order
is not key order) with two steps added:
  ("frame", cells)       UpdateReference() for a frame whose mvpMapPoints are `cells` (point indices, -1 = NULL)
  ("to_be_erased", kf)   SetNotErase() then SetBadFlag(): the keyframe gets mbToBeErased and stays live
Neither changes the map the model holds.  Besides its frame steps, every scene is probed after each step with
probe_frame(): every third point made so far, and point 0 at two cells."""
import numpy as np

import kf_culling_scenes as KS


class LmScene(KS.CullScene):
    def frame(self, cells):
        self.steps.append(("frame", np.asarray(cells, np.int32)))

    def to_be_erased(self, kf):
        self.steps.append(("to_be_erased", int(kf)))


class LmModel(KS.CullModel):
    def apply(self, step, erased=()):
        if step[0] in ("frame", "to_be_erased"):
            return
        super().apply(step, erased)


def probe_frame(model):
    n = len(model.obs)
    return np.array(([0, -1, 0] if n else [-1]) + list(range(0, n, 3)), np.int32)


def scene_tie_and_double_vote():
    """a tie of maxima (the smaller key is mpReferenceKF), and one point at three cells whose triple vote beats a keyframe
    seen through two points (a single vote per point would make that keyframe the reference)"""
    s = LmScene("tie_double_vote", 32, seed=41)
    k0, x, y = s.kf(), s.kf(), s.kf()
    p = s.seen(1, [x])
    q = s.seen(1, [y, k0])
    r = s.seen(1, [y])
    s.update([k0, x, y])
    s.frame([p, q])                 # K0, x and y 1 each: K0
    s.frame([q, -1, p])
    s.frame([p, p, p, q, r])        # x 3, y 2, K0 1: x
    s.frame([r, p])                 # x 1, y 1: x
    return s


def scene_empty_and_bad():
    """frames whose counter is empty (NULL cells only, a bad point only, a point whose only observer is retired) and a bad
    point at a frame cell next to good ones"""
    s = LmScene("empty_bad", 32, seed=42)
    k0, a, b, c = s.kf(), s.kf(), s.kf(), s.kf()
    p = s.seen(4, [a, b, c])
    lone = s.seen(1, [c])
    s.seen(20, [a, b])
    s.update([k0, a, b, c])
    s.frame([])
    s.frame([-1, -1, -1])
    s.bad_pt(p)
    s.frame([p])
    s.frame([p, p + 1, -1, p, p + 2])
    s.erase_kf(c)
    s.frame([lone, -1])
    return s


def scene_bound(n0, name=None):
    """n0 keyframes counted (one frame point each), each with a neighbour of its own that is not counted: the extension
    stops before a visit once more than 80 are listed (79 -> 81, 80 -> 81, 81 and more -> none appended)"""
    s = LmScene(name or "bound%d" % n0, 32, seed=43 + n0)
    k0 = s.kf()
    cs = [s.kf() for _ in range(n0)]
    bs = [s.kf() for _ in range(n0)]
    fp = [s.seen(1, [c]) for c in cs]
    for c, b in zip(cs, bs):
        s.seen(15 + (c % 3), [b, c])
    s.update([k0] + bs + cs)
    s.frame(fp)
    s.frame(fp[::-1] + [-1])
    return s


def scene_listed_and_limits():
    """c1's first neighbour c2 is counted (listed in step 3), so its second, b, is appended; c2's first neighbour b was
    appended by the earlier visit, so its second, d, is; b's own neighbour e is never reached (appended entries are not
    visited).  A hub's first 10 neighbours are all counted and its 11th is not: nothing is appended for it."""
    s = LmScene("listed_limits", 320, seed=44)
    k0, c1, c2, b, d, e, hub = (s.kf() for _ in range(7))
    ns = [s.kf() for _ in range(11)]
    f1, f2, fh = s.seen(1, [c1]), s.seen(1, [c2]), s.seen(1, [hub])
    s.seen(20, [c1, c2])
    s.seen(16, [c1, b])
    s.seen(18, [c2, b])
    s.seen(15, [c2, d])
    s.seen(25, [b, e])
    fn = []
    for j, n in enumerate(ns):
        s.seen(30 - j, [hub, n])
        fn.append(s.seen(1, [n]))
    s.update([k0, e, d, b, c2, c1] + ns + [hub])
    s.frame([f1, f2])
    s.frame([fh] + fn[:10])
    s.frame([fh] + fn[:9])          # the 10th neighbour not counted: appended
    s.frame([f2, f1, fh])
    return s


def scene_stale():
    """c's first neighbour r was retired while c's map still names it (r's own update no longer saw c, so its SetBadFlag did
    not erase the connection): the stale entry is skipped and c's second neighbour appended; also a counted keyframe with
    mbToBeErased is listed"""
    s = LmScene("stale", 128, seed=45)
    k0, c, r, h1, h2, h3, t = (s.kf() for _ in range(7))
    p = s.seen(20, [c, r, h1, h2])
    q = s.seen(15, [c, r])
    s.seen(5, [r, h3])
    s.seen(17, [c, t])
    f = s.seen(1, [c])
    g = s.seen(1, [t])
    s.update([k0, h1, h2, h3, t, r, c])   # c: r 35, h2 20, h1 20 (the larger key first on a tie), t 17
    for j in range(20):
        s.ba_erase(r, p + j)
    for j in range(15):
        s.ba_erase(r, q + j)               # q: one observer left, bad
    s.update([r])                          # r: {h3: 5}; c's map keeps r
    s.frame([f])
    s.erase_kf(r)
    s.frame([f])
    s.frame([f, g])
    s.to_be_erased(t)
    s.frame([f, g, g])
    return s


def scene_rows():
    """points shared across rows, a point named twice in one row (listed once, at its first cell), a queued keyframe's row
    (not an observer, not listed) and points made bad"""
    s = LmScene("rows", 64, seed=46)
    k0, a, b = s.kf(), s.kf(), s.kf()
    sh = s.seen(10, [b, a])
    p = s.seen(3, [a, b, k0])
    s.observe(p, a, s.free[a])        # a names p again at a later feature
    s.free[a] += 1
    own = s.seen(5, [b])
    qk = s.kfq()
    s.row(qk, 0, own)
    s.row(qk, 1, sh)
    s.update([k0, a, b])
    s.frame([sh, own, p])
    s.bad_pt(sh + 1)
    s.frame([sh + 1, sh + 2, p, p])
    s.process(qk)
    s.update([qk])
    s.frame([own, own + 1])         # the processed keyframe is an observer of `own` now
    return s


def small_scenes():
    return [scene_tie_and_double_vote(), scene_empty_and_bad(), scene_bound(79), scene_bound(80), scene_bound(81), scene_bound(100),
            scene_listed_and_limits(), scene_stale(), scene_rows()]


def large_frames(model, slot_of, kf=1000, sizes=(300, 1000, 2000), seed=51):
    """frames on covis_scenes.scene_large's map: `size` matched points from keyframe kf's row and its neighbours' (by
    creation index), shuffled, some at two cells"""
    rng = np.random.default_rng(seed)
    out = []
    for n in sizes:
        pool = []
        for k in (kf, kf + 1, kf - 1, kf + 2):
            row = model.kf_mp[k, :model.nfeat[k]]
            pool += [int(v) for v in row if v >= 0 and not model.bad[v]]
        pool = list(dict.fromkeys(pool))
        cells = rng.permutation(np.array(pool[:n], np.int32))
        if n > 10:
            cells[-5:] = cells[:5]
        out.append(cells)
    return out
