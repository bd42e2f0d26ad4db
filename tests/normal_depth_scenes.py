"""Scripted maps for MapPoint::UpdateNormalAndDepth (src/MapPoint.cc:273-312) and a numpy restatement of the rule with the
wrong variants the tests name (numpy only; used by the CPU and GPU test files of orbfe_normal_and_depth).

A scene is a dict:
  scale_factor, nlevels      the extractor's, shared by every keyframe (scale table: the float chain of Frame.cc:90-103)
  kfs                        per keyframe: center (float32 [3]; the pose is R = I, t = -center, whose GetCameraCenter() is
                             center bit for bit), octaves (int32 [n] of its keypoints), bad
  points                     per map point: pos (float32 [3]), ref (reference keyframe), obs [(keyframe, feature index)] in
                             keyframe creation order (the reference's mObservations order when keyframes ascend in memory),
                             pos2 (None, or the position a later SetWorldPos gives it: the local-BA pass), bad
  variants                   the wrong variants whose results must differ from the rule's on this scene
"""
import numpy as np

VARIANTS = ("fma", "double_sum", "reversed", "tree", "double_inv_n", "float_norm", "skip_bad", "level_flip")
F32 = np.float32


def scale_table(scale_factor, nlevels):
    t = [F32(1.0)]
    for _ in range(1, nlevels):
        t.append(F32(t[-1] * F32(scale_factor)))
    return np.array(t, np.float32)


def _keyframes(rng, n, nfeat, nlevels, spread=4.0, bad_every=0):
    kfs = []
    for k in range(n):
        kfs.append(dict(center=(rng.standard_normal(3) * spread).astype(np.float32),
                        octaves=rng.integers(0, nlevels, nfeat).astype(np.int32),
                        bad=bool(bad_every) and k % bad_every == 1))
    return kfs


def _point(rng, kfs, nobs, ref=None, obs_ref=True, dist=(5.0, 40.0)):
    """A point observed by nobs distinct keyframes (creation order), the reference keyframe among them unless obs_ref is
    False."""
    ks = np.sort(rng.choice(len(kfs), nobs, replace=False))
    if ref is None:
        ref = int(ks[rng.integers(0, nobs)]) if obs_ref else int(rng.integers(0, len(kfs)))
        if not obs_ref:
            while ref in ks:
                ref = int(rng.integers(0, len(kfs)))
    d = rng.standard_normal(3)
    pos = (kfs[ref]["center"] + d / np.linalg.norm(d) * rng.uniform(*dist)).astype(np.float32)
    obs = [(int(k), int(rng.integers(0, len(kfs[k]["octaves"])))) for k in ks]
    return dict(pos=pos, ref=ref, obs=obs, pos2=None, bad=False)


def scene_counts(seed=1):
    """Points of 1, 31, 32, 33, 64, 65 and 1000 observations (chunk edges of the warp) over 1000 keyframes."""
    rng = np.random.default_rng(seed)
    kfs = _keyframes(rng, 1000, 16, 8)
    pts = [_point(rng, kfs, n) for n in (1, 31, 32, 33, 64, 65, 1000) for _ in range(3)]
    return dict(name="counts", scale_factor=1.2, nlevels=8, kfs=kfs, points=pts,
                variants=("fma", "double_sum", "reversed", "tree", "double_inv_n", "float_norm", "level_flip"))


def scene_bad_keyframes(seed=2):
    """Every third keyframe isBad(): the reference still counts their observations."""
    rng = np.random.default_rng(seed)
    kfs = _keyframes(rng, 60, 16, 8, bad_every=3)
    pts = [_point(rng, kfs, int(n)) for n in rng.integers(2, 50, 80)]
    return dict(name="bad_keyframes", scale_factor=1.2, nlevels=8, kfs=kfs, points=pts,
                variants=("fma", "double_sum", "reversed", "tree", "double_inv_n", "float_norm", "skip_bad", "level_flip"))


def scene_octaves(nlevels, scale_factor, seed=3):
    """Reference octaves 0 and nlevels - 1 only."""
    rng = np.random.default_rng(seed + nlevels)
    kfs = _keyframes(rng, 40, 8, nlevels)
    pts = []
    for i in range(60):
        p = _point(rng, kfs, int(rng.integers(2, 30)))
        r = p["ref"]
        idx = [j for k, j in p["obs"] if k == r][0]
        kfs[r]["octaves"][idx] = 0 if i % 2 == 0 else nlevels - 1
        pts.append(p)
    # two points may share a reference feature: the later setting wins, and both read it, so every reference octave is 0 or nlevels - 1
    v = ("fma", "double_sum", "reversed", "tree", "double_inv_n", "float_norm")
    return dict(name="octaves_L%d" % nlevels, scale_factor=scale_factor, nlevels=nlevels, kfs=kfs, points=pts,
                variants=v + (("level_flip",) if nlevels > 1 else ()))


def scene_degenerate(seed=4):
    """A point on its reference keyframe's camera centre, the reference keyframe not among its observations (dist 0, finite
    normal; the reference's observations[pRefKF] reads index 0); a point on an observer's camera centre (NaN normal); a
    bad map point (returns before writing)."""
    rng = np.random.default_rng(seed)
    kfs = _keyframes(rng, 30, 8, 8)
    on_ref = _point(rng, kfs, 6, obs_ref=False)
    on_ref["pos"] = kfs[on_ref["ref"]]["center"].copy()
    on_obs = _point(rng, kfs, 7)
    on_obs["pos"] = kfs[on_obs["obs"][3][0]]["center"].copy()
    bad = _point(rng, kfs, 5)
    bad["bad"] = True
    absent = _point(rng, kfs, 9, obs_ref=False)
    pts = [on_ref, on_obs, bad, absent] + [_point(rng, kfs, int(n)) for n in rng.integers(2, 20, 20)]
    return dict(name="degenerate", scale_factor=1.2, nlevels=8, kfs=kfs, points=pts,
                variants=("fma", "double_sum", "reversed", "tree", "float_norm", "level_flip"))


def scene_local_ba(seed=5):
    """LocalBundleAdjustment's recovery: every point gets SetWorldPos (a small move), then one batch."""
    rng = np.random.default_rng(seed)
    kfs = _keyframes(rng, 80, 32, 8)
    pts = [_point(rng, kfs, int(n)) for n in rng.integers(2, 80, 300)]
    for p in pts:
        p["pos2"] = (p["pos"] + rng.standard_normal(3) * 0.05).astype(np.float32)
    return dict(name="local_ba", scale_factor=1.2, nlevels=8, kfs=kfs, points=pts,
                variants=("fma", "double_sum", "reversed", "tree", "double_inv_n", "float_norm", "level_flip"))


def all_scenes():
    return [scene_counts(), scene_bad_keyframes(), scene_octaves(1, 1.2), scene_octaves(8, 1.2), scene_octaves(32, 1.1),
            scene_degenerate(), scene_local_ba()]


def final_pos(p):
    return p["pos"] if p["pos2"] is None else p["pos2"]


def host_arrays(scene):
    """The scene in the layout of orbfe_normal_and_depth: (world, ref_centers, ref_octave, group_ptr, obs_centers, obs_bad).
    A bad map point is an empty group.  The reference octave is that of the reference keyframe's observed keypoint, index 0
    where the reference keyframe does not observe the point."""
    kfs, pts = scene["kfs"], scene["points"]
    world = np.array([final_pos(p) for p in pts], np.float32).reshape(-1, 3)
    ref_c = np.array([kfs[p["ref"]]["center"] for p in pts], np.float32).reshape(-1, 3)
    ref_oct = np.array([kfs[p["ref"]]["octaves"][ref_index(p)] for p in pts], np.int32)
    gp = np.cumsum([0] + [0 if p["bad"] else len(p["obs"]) for p in pts]).astype(np.int32)
    oc = [kfs[k]["center"] for p in pts if not p["bad"] for k, _ in p["obs"]]
    ob = [kfs[k]["bad"] for p in pts if not p["bad"] for k, _ in p["obs"]]
    return world, ref_c, ref_oct, gp, np.array(oc, np.float32).reshape(-1, 3), np.array(ob, bool)


def ref_index(p):
    for k, j in p["obs"]:
        if k == p["ref"]:
            return j
    return 0


def _norm(d, variant):
    if variant == "float_norm":
        return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float64)
    dd = d.astype(np.float64)
    return np.sqrt((dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2])


def _tree32(t):
    """One butterfly reduction of a 32-lane chunk (lane 0's result), the order a warp shuffle reduction adds in."""
    v = np.zeros((32, 3), np.float32)
    v[:len(t)] = t
    lanes = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        v = (v + v[lanes ^ off]).astype(np.float32)
    return v[0]


def restate(world, ref_c, ref_oct, gp, oc, obs_bad, scale_factor, sfs, variant=None, normal=None, min_dist=None, max_dist=None):
    """The rule of DESIGN.md §2 in numpy, or one named wrong variant of it.  Returns (normal, min_dist, max_dist) float32."""
    n_pts = len(gp) - 1
    out_n = np.zeros((n_pts, 3), np.float32) if normal is None else np.array(normal, np.float32, copy=True)
    out_a = np.zeros(n_pts, np.float32) if min_dist is None else np.array(min_dist, np.float32, copy=True)
    out_b = np.zeros(n_pts, np.float32) if max_dist is None else np.array(max_dist, np.float32, copy=True)
    sf, nl = F32(scale_factor), len(sfs)
    with np.errstate(all="ignore"):
        for g in range(n_pts):
            b, e = int(gp[g]), int(gp[g + 1])
            if e <= b:
                continue
            P = world[g]
            C = oc[b:e]
            if variant == "skip_bad":
                C = C[~obs_bad[b:e]]
            d = (P[None, :] - C).astype(np.float32)
            a = (1.0 / _norm(d, variant)).astype(np.float32)
            if variant == "fma":
                acc = np.zeros(3, np.float32)
                for j in range(len(d)):
                    acc = (d[j].astype(np.float64) * np.float64(a[j]) + acc.astype(np.float64)).astype(np.float32)
            else:
                t = (d * a[:, None]).astype(np.float32)
                if variant == "double_sum":
                    acc = np.add.accumulate(np.vstack([np.zeros((1, 3)), t.astype(np.float64)]), axis=0)[-1].astype(np.float32)
                elif variant == "tree":
                    acc = np.zeros(3, np.float32)
                    for c0 in range(0, len(t), 32):
                        acc = (acc + _tree32(t[c0:c0 + 32])).astype(np.float32)
                else:
                    tt = t[::-1] if variant == "reversed" else t
                    acc = np.add.accumulate(np.vstack([np.zeros((1, 3), np.float32), tt]), axis=0, dtype=np.float32)[-1]
            n = len(d)
            if variant == "double_inv_n":
                out_n[g] = (acc.astype(np.float64) * (np.float64(1.0) / n)).astype(np.float32) + F32(0.0)
            else:
                out_n[g] = (acc * F32(np.float64(1.0) / n)).astype(np.float32) + F32(0.0)
            pc = (P - ref_c[g]).astype(np.float32)
            dist = F32(_norm(pc[None, :], variant)[0])
            lvl = int(ref_oct[g])
            out_a[g] = F32(F32(F32(F32(1.0) / sf) * dist) / sfs[lvl])
            out_b[g] = F32(F32(sf * dist) * sfs[lvl if variant == "level_flip" else nl - 1 - lvl])
    return out_n, out_a, out_b


def same(x, y):
    """Bit equality with every NaN equal to every NaN."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    if x.shape != y.shape:
        return False
    nx, ny = np.isnan(x), np.isnan(y)
    return bool(np.array_equal(nx, ny) and np.array_equal(x.view(np.uint32)[~nx], y.view(np.uint32)[~ny]))


def frame_store(scene, cap=None):
    """The scene as a frame store for orbfe_normal_and_depth_device: (kps [nframes*cap] octaves, counts, centers [nframes,3],
    group_ptr, obs slots, ref slots, world).  Frame row f = keyframe f, slot = f*cap + feature index."""
    kfs, pts = scene["kfs"], scene["points"]
    cap = cap or max(len(k["octaves"]) for k in kfs)
    octs = np.zeros(len(kfs) * cap, np.int32)
    for f, k in enumerate(kfs):
        octs[f * cap:f * cap + len(k["octaves"])] = k["octaves"]
    counts = np.array([len(k["octaves"]) for k in kfs], np.int32)
    centers = np.array([k["center"] for k in kfs], np.float32)
    gp = np.cumsum([0] + [0 if p["bad"] else len(p["obs"]) for p in pts]).astype(np.int32)
    obs = np.array([k * cap + j for p in pts if not p["bad"] for k, j in p["obs"]], np.int32)
    ref = np.array([p["ref"] * cap + ref_index(p) for p in pts], np.int32)
    world = np.array([final_pos(p) for p in pts], np.float32).reshape(-1, 3)
    return octs, counts, centers, gp, obs, ref, world, cap
