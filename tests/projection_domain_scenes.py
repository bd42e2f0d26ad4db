"""Scenes for the projecting matchers at their rounding edges (numpy only).

The projecting matchers start with float arithmetic: each map point is projected (`x3Dc = Rcw*x3Dw + tcw` as OpenCV's small
`gemm`, `invzc = 1.0/zc`, `u = fx*xc*invzc + cx`), tested against the image bounds, turned into a cell range of Frame's grid
and a window `|kp.x - u| > r`.  SearchByProjection(Frame, KeyFrame) also predicts the level from `dist3D / minDistance`, the
local-map search picks its radius from the viewing cosine, and SearchForTriangulation tests the epipolar distance.  This
module restates that geometry with every binary32 operation rounded once, in the reference's order, and builds scenes with
general poses (rotations that are not multiples of 90 degrees), TUM-like intrinsics (fx != fy, non-integer cx, cy), depths
0.5-50 and scale factors 1.2 x 8 and 1.5 x 12 whose points sit on one of those decisions: found by a bounded search over
float32 inputs (a world coordinate or a keypoint moved ulp by ulp).

Each scene keeps its facts (which decision a query sits on and on which side, as the restatement decides it) and the
wrong variants that change its matches (`VARIANTS`).  A variant is a one-line change of the restatement:

- `fma_gemm`: the gemm row as fma(r2, x2, fma(r1, x1, r0*x0)); `double_gemm`: the row summed in double; `gemm_reversed`:
  (r2*x2 + r1*x1) + r0*x0;
- `assoc_uv`: fx*(xc*invzc); `fma_uv`: fma(fx*xc, invzc, cx); `divide_uv`: fx*(xc/zc);
- `bounds_inclusive`: a projection on a bound is dropped; `window_ge`: a candidate at |dx| == r is dropped;
- `radius_pow`: the scale table from powf instead of Frame.cc's product chain; `upper_bound`: a ratio equal to a scale
  factor predicts the next level; `float_norm`: dist3D summed and rooted in float;
- `view_cos_float`: RadiusByViewingCos compares with 0.998f instead of the double 0.998;
- `fma_line`: each line coefficient as fma(y1, F3, x1*F0) + F6; `line_reordered`: x1*F0 + (y1*F3 + F6); `fma_num`:
  fma(lb, y2, la*x2) + lc; `float_thr`: dsqr < 3.84f*sigma2 in float.

The fused multiply-adds are emulated: the exact product in double, one addition in double, one rounding to float.  Two
changes a CPU probe found equal to the rule on 200,000 random projections -- adding t in float instead of through double,
and 1.0f/zc -- are not variants: no scene here separates them.

The cell range of GetFeaturesInArea has no scene of its own.  Frame's grid assigns a keypoint to `round((x - minX) *
gridInv)`, so every keypoint of the cell that a floor / ceil edge adds or removes lies at least half a cell outside the
window `|kp.x - u| <= r`: no rounding of the cell range can change a match, and the window test is what the window scenes
pin.

All keypoint angles are 0, so the rotation histogram keeps every match; the restatement leaves it out."""
import numpy as np

F32, F64 = np.float32, np.float64
KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])

# TUM fr1-like intrinsics, 640 x 480, zero distortion: bounds (0, 0, 640, 480), gridInv = 64/640 = 48/480 = 0.1f (not exact)
FX, FY, CX, CY = F32(517.3), F32(516.5), F32(318.6), F32(255.3)
W, H = 640, 480
BOUNDS = (F32(0), F32(0), F32(W), F32(H))
GINV = (F32(64) / F32(W), F32(48) / F32(H))
TH_HIGH = 100

PROJ_VARIANTS = ["fma_gemm", "double_gemm", "gemm_reversed", "assoc_uv", "fma_uv", "divide_uv"]
VARIANTS_BY_ROUTINE = {
    "ff": PROJ_VARIANTS + ["bounds_inclusive", "window_ge", "radius_pow"],
    "kf": PROJ_VARIANTS + ["bounds_inclusive", "window_ge", "radius_pow", "upper_bound", "float_norm"],
    "f1f2": PROJ_VARIANTS + ["window_ge"],
    "local": ["window_ge", "radius_pow", "view_cos_float"],
    "tri": ["fma_line", "line_reordered", "fma_num", "float_thr"],
}
ALL_VARIANTS = sorted({v for vs in VARIANTS_BY_ROUTINE.values() for v in vs})


# ---- float32 helpers ------------------------------------------------------------------------------------------------------
def fma(a, b, c):
    """fmaf emulated: the exact product in double, one double addition, one rounding to float"""
    return (np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64) + np.asarray(c, F32).astype(F64)).astype(F32)


def _ordered(x):
    i = np.asarray(x, F32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def steps(x, ks):
    """the floats ks ulps away from x (ks an int array)"""
    o = _ordered(x) + np.asarray(ks, np.int64)
    return np.where(o < 0, (-o) | 0x80000000, o).astype(np.uint32).view(F32)


def next_up(x):
    return F32(np.nextafter(F32(x), F32(np.inf)))


def next_down(x):
    return F32(np.nextafter(F32(x), F32(-np.inf)))


def rotation(axis, deg):
    """Rodrigues' rotation in double, rounded to float once"""
    k = np.asarray(axis, F64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    th = np.deg2rad(deg)
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def pose(axis, deg, t):
    T = np.zeros((3, 4), F64)
    T[:, :3], T[:, 3] = rotation(axis, deg), t
    return T.astype(F32)


POSES = {
    "a": pose((0.3, -0.8, 0.5), 7.0, (0.13, -0.07, 0.21)),
    "b": pose((-0.6, 0.2, 0.77), 23.0, (-0.4, 0.25, 1.3)),
    "c": pose((0.1, 0.9, -0.4), 41.0, (1.7, -0.9, 0.35)),
}
SCALES = {"1.2x8": (1.2, 8), "1.5x12": (1.5, 12)}


def scale_table(scale, nlevels, variant=None):
    """Frame.cc's mvScaleFactors: sf[i] = sf[i-1] * scale in float; `radius_pow`: powf(scale, i)"""
    s = F32(scale)
    if variant == "radius_pow":
        return np.array([F32(F64(s) ** i) for i in range(nlevels)], F32)
    sf = [F32(1)]
    for _ in range(1, nlevels):
        sf.append(F32(sf[-1] * s))
    return np.array(sf, F32)


def sigma2(scale, nlevels):
    sf = scale_table(scale, nlevels)
    return (sf * sf).astype(F32)


# ---- the restatement ------------------------------------------------------------------------------------------------------
def camera_point(T, X, variant=None):
    """x3Dc = Rcw*x3Dw + tcw, OpenCV's small gemm: the three products summed in float left to right, then
    (float)((double)sum + (double)t)"""
    X = np.atleast_2d(np.asarray(X, F32))
    x0, x1, x2 = X[:, 0], X[:, 1], X[:, 2]
    out = []
    for k in range(3):
        r0, r1, r2, t = (F32(T[k, j]) for j in range(4))
        if variant == "double_gemm":
            s = F64(r0) * x0.astype(F64) + F64(r1) * x1.astype(F64) + F64(r2) * x2.astype(F64)
        elif variant == "fma_gemm":
            s = fma(r2, x2, fma(r1, x1, r0 * x0))
        elif variant == "gemm_reversed":
            s = (r2 * x2 + r1 * x1) + r0 * x0
        else:
            s = (r0 * x0 + r1 * x1) + r2 * x2
        out.append((np.asarray(s).astype(F64) + F64(t)).astype(F32))
    return out


def project(T, X, variant=None):
    """(u, v) of SearchByProjection: invzc = (float)(1.0/(double)zc), u = ((fx*xc)*invzc) + cx"""
    xc, yc, zc = camera_point(T, X, variant)
    invzc = (1.0 / zc.astype(F64)).astype(F32)
    if variant == "assoc_uv":
        return FX * (xc * invzc) + CX, FY * (yc * invzc) + CY
    if variant == "fma_uv":
        return fma(FX * xc, invzc, CX), fma(FY * yc, invzc, CY)
    if variant == "divide_uv":
        return FX * (xc / zc) + CX, FY * (yc / zc) + CY
    return (FX * xc) * invzc + CX, (FY * yc) * invzc + CY


def in_bounds(u, v, variant=None):
    """`u < mnMinX || u > mnMaxX` (and v) drops the point"""
    if variant == "bounds_inclusive":
        return (u > BOUNDS[0]) & (u < BOUNDS[2]) & (v > BOUNDS[1]) & (v < BOUNDS[3])
    return ~((u < BOUNDS[0]) | (u > BOUNDS[2]) | (v < BOUNDS[1]) | (v > BOUNDS[3]))


def camera_centre(T):
    """Ow = -Rcw.t()*tcw: gemm's general path, double accumulation, times -1"""
    T64 = T.astype(F64)
    return np.array([(T64[0, k] * T64[0, 3] + T64[1, k] * T64[1, 3] + T64[2, k] * T64[2, 3]) * -1.0 for k in range(3)]).astype(F32)


def dist3d(T, X, variant=None):
    """cv::norm(x3Dw - Ow): the float differences, the squares summed in double, sqrt in double, rounded to float"""
    PO = np.atleast_2d(np.asarray(X, F32)) - camera_centre(T)
    if variant == "float_norm":
        return np.sqrt((PO[:, 0] * PO[:, 0] + PO[:, 1] * PO[:, 1]) + PO[:, 2] * PO[:, 2])
    P = PO.astype(F64)
    return np.sqrt(P[:, 0] * P[:, 0] + P[:, 1] * P[:, 1] + P[:, 2] * P[:, 2]).astype(F32)


def predicted_level(ratio, sf, variant=None):
    """lower_bound(mvScaleFactors, ratio), clamped to nlevels - 1; `upper_bound`: the first factor above ratio"""
    it = int(np.sum(sf <= ratio)) if variant == "upper_bound" else int(np.sum(sf < ratio))
    return min(it, len(sf) - 1)


def view_radius(view_cos, variant=None):
    """RadiusByViewingCos: a float cosine compared with the double 0.998"""
    if variant == "view_cos_float":
        return F32(2.5) if F32(view_cos) > F32(0.998) else F32(4.0)
    return F32(2.5) if F64(F32(view_cos)) > 0.998 else F32(4.0)


def window_ok(kx, ky, u, v, r, variant=None):
    dx, dy = np.abs(F32(kx) - F32(u)), np.abs(F32(ky) - F32(v))
    if variant == "window_ge":
        return not (dx >= r or dy >= r)
    return not (dx > r or dy > r)


def epipolar(x1, y1, x2, y2, F, sig2, variant=None):
    """CheckDistEpipolarLine: the line x1' F12, num, den, dsqr = num*num/den; (double)dsqr < 3.84*(double)sigma2.
    Returns (ok, dsqr)."""
    x1, y1, x2, y2 = F32(x1), F32(y1), F32(x2), F32(y2)
    F = np.asarray(F, F32).reshape(-1)

    def line(a, b, c):
        if variant == "fma_line":
            return fma(y1, b, x1 * a) + c
        if variant == "line_reordered":
            return x1 * a + (y1 * b + c)
        return (x1 * a + y1 * b) + c
    la, lb, lc = line(F[0], F[3], F[6]), line(F[1], F[4], F[7]), line(F[2], F[5], F[8])
    num = fma(lb, y2, la * x2) + lc if variant == "fma_num" else (la * x2 + lb * y2) + lc
    den = la * la + lb * lb
    if den == 0:
        return False, F32(np.nan)
    dsqr = F32(num * num) / den
    if variant == "float_thr":
        return bool(dsqr < F32(F32(3.84) * F32(sig2))), dsqr
    return bool(F64(dsqr) < 3.84 * F64(F32(sig2))), dsqr


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


class Frame:
    """The slice of Frame the matchers read, with Frame's grid: round((x - minX) * gridInv), push_back order"""

    def __init__(self, kps, desc, scale, nlevels, variant=None):
        self.kps, self.desc = kps, desc
        self.sf = scale_table(scale, nlevels, variant)
        self.cell = {}
        for i, k in enumerate(kps):
            a = F32(F32(k["x"] - BOUNDS[0]) * GINV[0])
            b = F32(F32(k["y"] - BOUNDS[1]) * GINV[1])
            px, py = int(np.sign(a) * np.floor(abs(F64(a)) + 0.5)), int(np.sign(b) * np.floor(abs(F64(b)) + 0.5))
            if 0 <= px < 64 and 0 <= py < 48:
                self.cell.setdefault((px, py), []).append(i)

    def features_in_area(self, u, v, r, lo, hi, variant=None):
        """GetFeaturesInArea: floor / ceil of the float window edges times gridInv, ix outer, iy inner, then the levels and
        the window test"""
        x0 = max(0, int(np.floor(F32(F32(F32(u) - BOUNDS[0]) - r) * GINV[0])))
        x1 = min(63, int(np.ceil(F32(F32(F32(u) - BOUNDS[0]) + r) * GINV[0])))
        y0 = max(0, int(np.floor(F32(F32(F32(v) - BOUNDS[1]) - r) * GINV[1])))
        y1 = min(47, int(np.ceil(F32(F32(F32(v) - BOUNDS[1]) + r) * GINV[1])))
        if x0 >= 64 or x1 < 0 or y0 >= 48 or y1 < 0:
            return []
        out = []
        for ix in range(x0, x1 + 1):
            for iy in range(y0, y1 + 1):
                for i in self.cell.get((ix, iy), []):
                    o = int(self.kps[i]["octave"])
                    if not (lo == -1 and hi == -1):
                        if (lo == hi and o != lo) or (lo != hi and (o < lo or o > hi)):
                            continue
                    if window_ok(self.kps[i]["x"], self.kps[i]["y"], u, v, r, variant):
                        out.append(i)
        return out


def guided(fr, queries, rule, nnratio, th_dist, variant=None):
    """The sequential loop of the projecting matchers over (u, v, r, lo, hi, desc, owner) queries: candidates whose slot is
    free, strict-< best and second best; rule 0 best <= th_dist (:1576, :1693); rule 1 best <= second*nnratio && best <=
    TH_HIGH (:586); rule 2 best <= TH_HIGH && !(same level && best > nnratio*second) (:113-121)."""
    slot = np.full(len(fr.kps), -1, np.int32)
    nm = 0
    for u, v, r, lo, hi, d, owner in queries:
        best, best2, bi, bl, bl2 = 2 ** 31 - 1, 2 ** 31 - 1, -1, -1, -1
        for i in fr.features_in_area(u, v, r, lo, hi, variant):
            if slot[i] >= 0:
                continue
            dist = hamming(d, fr.desc[i])
            if dist < best:
                best2, bl2, best, bl, bi = best, bl, dist, int(fr.kps[i]["octave"]), i
            elif dist < best2:
                best2, bl2 = dist, int(fr.kps[i]["octave"])
        if rule == 0:
            ok = best <= th_dist
        elif rule == 1:
            ok = F32(best) <= F32(best2) * F32(nnratio) and best <= TH_HIGH
        else:
            ok = best <= TH_HIGH and not (bl == bl2 and F32(best) > F32(nnratio) * F32(best2))
        if ok:
            slot[bi] = owner
            nm += 1
    return nm, slot


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def descriptors(n, offset=0):
    """rows of the 256 x 256 Sylvester-Hadamard matrix as bits: any two are 128 apart, above TH_HIGH"""
    Hm = np.array([[1]])
    while Hm.shape[0] < 256:
        Hm = np.block([[Hm, Hm], [Hm, -Hm]])
    assert offset + n <= 256
    return np.packbits((Hm[offset:offset + n] > 0).astype(np.uint8), axis=1)


def keypoints(xy, octaves):
    k = np.zeros(len(xy), KP_DTYPE)
    if len(xy):
        xy = np.asarray(xy, F32).reshape(-1, 2)
        k["x"], k["y"] = xy[:, 0], xy[:, 1]
    k["octave"] = octaves
    k["size"], k["response"] = 31.0, 1.0
    return k


class Scene:
    """One routine's inputs.  `facts`: (query, label, matched) -- the decision each query sits on and whether the
    restatement matches it; `variants`: the variants that change the scene's matches."""

    def __init__(self, name, routine, **kw):
        self.name, self.routine = name, routine
        self.__dict__.update(kw)
        self.facts = []

    def run(self, variant=None):
        return RUN[self.routine](self, variant)

    @property
    def variants(self):
        return set(VARIANTS[self.name])


def _run_ff(s, variant):
    cur = Frame(s.cur_kps, s.cur_desc, s.scale, s.nlevels, variant)
    u, v = project(s.T, s.world, variant)
    keep = in_bounds(u, v, variant)
    Q = []
    for i in range(len(s.world)):
        if keep[i]:
            o = int(s.last_kps[i]["octave"])
            Q.append((u[i], v[i], F32(s.th) * cur.sf[o], o - 1, o + 1, s.last_desc[i], i))
    return guided(cur, Q, 0, 0.0, TH_HIGH, variant)


def _run_kf(s, variant):
    cur = Frame(s.cur_kps, s.cur_desc, s.scale, s.nlevels, variant)
    u, v = project(s.T, s.world, variant)
    keep = in_bounds(u, v, variant)
    d3 = dist3d(s.T, s.world, variant)
    Q = []
    for i in range(len(s.world)):
        if keep[i]:
            lv = predicted_level(F32(d3[i] / s.min_dist[i]), cur.sf, variant)
            Q.append((u[i], v[i], F32(s.th) * cur.sf[lv], lv - 1, lv + 1, s.desc[i], i))
    return guided(cur, Q, 0, 0.0, s.orb_dist, variant)


def _run_f1f2(s, variant):
    f2 = Frame(s.f2_kps, s.f2_desc, s.scale, s.nlevels, variant)
    u, v = project(s.T, s.world, variant)
    Q = [(u[i], v[i], F32(s.window), int(s.f1_kps[i]["octave"]), int(s.f1_kps[i]["octave"]), s.f1_desc[i], i)
         for i in range(len(s.world))]
    return guided(f2, Q, 1, s.nnratio, TH_HIGH, variant)


def _run_local(s, variant):
    f = Frame(s.kps, s.desc, s.scale, s.nlevels, variant)
    Q = []
    for i in range(len(s.proj)):
        r = view_radius(s.view_cos[i], variant)
        if F32(s.th) != F32(1):
            r = F32(r * F32(s.th))
        lv = int(s.level[i])
        Q.append((s.proj[i, 0], s.proj[i, 1], F32(r * f.sf[lv]), lv - 1, lv, s.mp_desc[i], i))
    return guided(f, Q, 2, s.nnratio, TH_HIGH, variant)


def _run_tri(s, variant):
    """SearchForTriangulation on one common node holding every feature (no side has map points): per side-1 feature the free
    side-2 candidates with distance <= TH_LOW, by (distance, index), the first within round(2 * best) that passes the epipolar
    test"""
    m12 = np.full(len(s.k1), -1, np.int32)
    matched = np.zeros(len(s.k2), bool)
    nm = 0
    for i1 in range(len(s.k1)):
        c = sorted((hamming(s.d1[i1], s.d2[i2]), i2) for i2 in range(len(s.k2)) if not matched[i2])
        c = [(d, i2) for d, i2 in c if d <= 50]
        if not c:
            continue
        for d, i2 in c:
            if d > round(2.0 * c[0][0]):
                break
            if epipolar(s.k1[i1]["x"], s.k1[i1]["y"], s.k2[i2]["x"], s.k2[i2]["y"], s.F12, s.sig2[s.k2[i2]["octave"]], variant)[0]:
                m12[i1], matched[i2] = i2, True
                nm += 1
                break
    return nm, m12


RUN = {"ff": _run_ff, "kf": _run_kf, "f1f2": _run_f1f2, "local": _run_local, "tri": _run_tri}


def changes(scene, variant):
    a, b = scene.run(), scene.run(variant)
    return a[0] != b[0] or not np.array_equal(a[1], b[1])


def _backproject(T, u, v, z):
    """a world point that projects near (u, v) at depth z (double, rounded to float)"""
    Xc = np.array([(u - float(CX)) / float(FX) * z, (v - float(CY)) / float(FY) * z, z])
    T64 = T.astype(F64)
    return (T64[:, :3].T @ (Xc - T64[:, 3])).astype(F32)


def _proj_changes(T, X, axis):
    """the projection variants that move u (axis 0) or v (axis 1) of X"""
    base = project(T, X)[axis][0]
    return {var for var in PROJ_VARIANTS if project(T, X, var)[axis][0] != base}


# bounds: (name, axis, bound value, outward direction)
SIDES = [("minX", 0, BOUNDS[0], -1), ("maxX", 0, BOUNDS[2], 1), ("minY", 1, BOUNDS[1], -1), ("maxY", 1, BOUNDS[3], 1)]


def _bound_pair(T, side, rng):
    """A world point whose projection lies exactly on the bound and one whose projection is the first value outside it
    that the walk reaches (u = fx*xc*invzc + cx is a multiple of ulp(cx) near 0, so next to bound 0 that is the next
    multiple, not the next float), found by walking one world coordinate ulp by ulp from a back-projected start"""
    name, axis, b, out = side
    for _ in range(200):
        z = rng.uniform(0.5, 50)
        other = rng.uniform(60, (H if axis == 0 else W) - 60)
        X = _backproject(T, float(b), other, z) if axis == 0 else _backproject(T, other, float(b), z)
        for j in np.argsort(-np.abs(T[axis, :3].astype(F64) * np.abs(X.astype(F64)))):
            ks = np.arange(-2000, 2001)
            cand = np.repeat(X[None], len(ks), 0)
            cand[:, j] = steps(X[j], ks)
            val = project(T, cand)[axis]
            on, off = np.flatnonzero(val == b), np.flatnonzero(val * out > b * out)
            if len(on) and len(off):
                first = val[off].min() if out > 0 else val[off].max()
                if first == steps(b, out) or b == 0:
                    return cand[on[0]], cand[off[np.flatnonzero(val[off] == first)[0]]]
    raise AssertionError("no point on bound %s" % name)


def _candidate_near(u, v, r, axis, out):
    """a Current keypoint 0.75 r inside the bound from (u, v): in the window, on the grid"""
    d = F32(0.75) * F32(r)
    return (F32(u - out * d), F32(v)) if axis == 0 else (F32(u), F32(v - out * d))


def bounds_scene(routine, pose_name, scale_name, seed):
    """Per image bound: map points projecting exactly on it (kept) and on the next float outside (dropped), each with its
    own candidate 0.75 r inside; extra pairs are added until every projection variant moves one of them."""
    T, (scale, nl) = POSES[pose_name], SCALES[scale_name]
    rng = np.random.default_rng(seed)
    sf = scale_table(scale, nl)
    th, oct_ = window_th(scale, nl), 1
    r = F32(F32(th) * sf[oct_])
    pts, kind = [], []
    need = set(PROJ_VARIANTS)
    tries = 0
    while tries < 4 or (need and tries < 60):
        side = SIDES[tries % 4]
        on, off = _bound_pair(T, side, rng)
        got = _proj_changes(T, on, side[1]) | _proj_changes(T, off, side[1])
        if tries < 4 or got & need:
            pts += [on, off]
            kind += [(side, True), (side, False)]
            need -= got
        tries += 1
    assert not need, need
    world = np.array(pts, F32)
    u, v = project(T, world)
    n = len(world)
    xy = [_candidate_near(u[i], v[i], r, s[1], s[3]) for i, (s, _) in enumerate(kind)]
    desc = descriptors(n)
    kw = dict(T=T, world=world, th=th, scale=scale, nlevels=nl)
    if routine == "ff":
        sc = Scene("%s-bounds-%s-%s" % (routine, pose_name, scale_name), "ff", cur_kps=keypoints(xy, oct_), cur_desc=desc,
                   last_kps=keypoints(np.zeros((n, 2)), oct_), last_desc=desc, **kw)
    else:   # minDistance puts the predicted level well inside level oct_
        md = (dist3d(T, world).astype(F64) / ((sf[oct_ - 1] + sf[oct_]) / 2.0)).astype(F32)
        sc = Scene("%s-bounds-%s-%s" % (routine, pose_name, scale_name), "kf", cur_kps=keypoints(xy, oct_), cur_desc=desc,
                   desc=desc, min_dist=md, orb_dist=TH_HIGH, **kw)
    for i, (s, on) in enumerate(kind):
        sc.facts.append((i, "%s %s" % ("on" if on else "next float outside", s[0]), on))
    return sc


def _window_candidates(u, r):
    """keypoint coordinates k with float(k - u) == r and == -r (at the window edge), and the first floats beyond them"""
    res = {}
    for sgn in (1, -1):
        ks = steps(F32(u + sgn * r), np.arange(-64, 65))
        d = (ks - F32(u)) * sgn
        at = np.flatnonzero(d == r)
        beyond = np.flatnonzero(d > r)
        if not len(at):
            return None
        res[sgn] = (ks[at[0]], ks[beyond[0]] if sgn == 1 else ks[beyond[-1]])
    return res


def _window_queries(u, v, r):
    """8 candidate positions around (u, v): at |dx| == r and one float beyond, both signs, both axes; None if an edge float
    does not exist for this (u, v, r)"""
    cx_, cy_ = _window_candidates(u, r), _window_candidates(v, r)
    if cx_ is None or cy_ is None:
        return None
    out = []
    for sgn in (1, -1):
        for j, lab in enumerate(("at r", "beyond r")):
            out.append(((cx_[sgn][j], F32(v)), "%s dx %s" % (lab, "+" if sgn > 0 else "-"), j == 0))
            out.append(((F32(u), cy_[sgn][j]), "%s dy %s" % (lab, "+" if sgn > 0 else "-"), j == 0))
    return out


def _pow_level(scale, nl, lo=1):
    """the first level >= lo whose powf factor differs from Frame's product chain (lo if none does: every power of 1.5 up
    to 1.5^11 is exact in float, so for 1.5 the two tables are equal)"""
    a, b = scale_table(scale, nl), scale_table(scale, nl, "radius_pow")
    return next((l for l in range(lo, nl) if a[l] != b[l]), lo)


def window_th(scale, nl):
    """th of the window scenes (r = th * sf[level] about 17 px); the bounds scenes of the same scale use it too, so that
    SearchByProjection(Frame, Frame) runs them in one launch"""
    return float(17.0 / float(scale_table(scale, nl)[_pow_level(scale, nl)]))


def window_scene(routine, pose_name, scale_name, seed):
    """Projections (u, v) in [20, 32) (where a window edge |kp - u| == r is a float) with eight candidates each, at r and
    one float beyond; projections are added until every projection variant moves one of them.  The window r is
    th * sf[level] at a level whose powf factor differs (SearchByProjection(F1, F2): the integer window)."""
    T, (scale, nl) = POSES[pose_name], SCALES[scale_name]
    rng = np.random.default_rng(seed)
    sf = scale_table(scale, nl)
    lev = _pow_level(scale, nl)
    th = 10.0
    r = F32(20) if routine == "f1f2" else F32(F32(th) * sf[lev])
    if routine != "f1f2":   # keep 16 <= r < 20 so that u - r stays on the grid
        th = window_th(scale, nl)
        r = F32(F32(th) * sf[lev])
    pts, qs = [], []
    need = set(PROJ_VARIANTS)
    tries = 0
    while (tries < 2 or need) and tries < 400:
        tries += 1
        X = _backproject(T, rng.uniform(21, 31), rng.uniform(21, 31), rng.uniform(0.5, 50))
        u, v = project(T, X)
        if not (20 <= u[0] < 32 and 20 <= v[0] < 32):
            continue
        q = _window_queries(u[0], v[0], r)
        if q is None:
            continue
        got = _proj_changes(T, X, 0) | _proj_changes(T, X, 1)
        if len(pts) < 2 or got & need:
            pts.append(X)
            qs.append(q)
            need -= got
    assert not need, need
    world = np.array([X for X, q in zip(pts, qs) for _ in q], F32)
    xy = [c for q in qs for c, _, _ in q]
    n = len(world)
    desc = descriptors(n)
    name = "%s-window-%s-%s" % (routine, pose_name, scale_name)
    kw = dict(T=T, world=world, scale=scale, nlevels=nl)
    if routine == "ff":
        sc = Scene(name, "ff", cur_kps=keypoints(xy, lev), cur_desc=desc, last_kps=keypoints(np.zeros((n, 2)), lev),
                   last_desc=desc, th=th, **kw)
    elif routine == "kf":
        md = (dist3d(T, world).astype(F64) / ((sf[lev - 1] + sf[lev]) / 2.0)).astype(F32)
        sc = Scene(name, "kf", cur_kps=keypoints(xy, lev), cur_desc=desc, desc=desc, min_dist=md, th=th, orb_dist=TH_HIGH, **kw)
    else:
        sc = Scene(name, "f1f2", f1_kps=keypoints(np.zeros((n, 2)), 2), f1_desc=desc, f2_kps=keypoints(xy, 2), f2_desc=desc,
                   window=int(r), nnratio=0.9, **kw)
    i = 0
    for q in qs:
        for _, lab, kept in q:
            sc.facts.append((i, lab, kept))
            i += 1
    return sc


def level_scene(pose_name, scale_name, seed):
    """SearchByProjection(Frame, KeyFrame): for every level l, minDistance such that ratio = dist3D/minDistance is exactly
    sf[l], one float below and one float above; a ratio below 1 and one above sf[n-1].  The candidate sits at octave l-1
    at the projection (found at level l, lost at level l+1); for l = 0 at octave 0 between th and th*sf[1] from it (found
    only at level 1).  One world point per level is chosen where dist3D in float differs upwards."""
    T, (scale, nl) = POSES[pose_name], SCALES[scale_name]
    rng = np.random.default_rng(seed)
    sf = scale_table(scale, nl)
    th = 6.0
    world, md, xy, octs, facts = [], [], [], [], []

    def ratio_md(X, target):
        """a minDistance with float(dist3D / minDistance) == target"""
        d = dist3d(T, X)[0]
        m = steps(F32(F64(d) / F64(target)), np.arange(-8, 9))
        hit = np.flatnonzero((d / m).astype(F32) == target)
        return m[hit[0]] if len(hit) else None

    def add(X, target, lv, label, matched):
        """a map point at X with ratio `target` and the candidate of level lv"""
        m = ratio_md(X, target)
        assert m is not None, label
        u, v = project(T, X)
        if lv == 0:
            d = F32(F32(th) * (F32(1) + sf[1]) / F32(2))
            xy.append((F32(u[0] + d), v[0]))
            octs.append(0)
        else:
            xy.append((u[0], v[0]))
            octs.append(lv - 1)
        world.append(X)
        md.append(m)
        facts.append((len(world) - 1, label, matched))

    for l in range(nl):
        best = None
        for _ in range(400):
            X = _backproject(T, rng.uniform(100, 540), rng.uniform(100, 380), rng.uniform(0.5, 50))
            if ratio_md(X, sf[l]) is None or ratio_md(X, next_up(sf[l])) is None or ratio_md(X, next_down(sf[l])) is None:
                continue
            best = best if best is not None else X
            if dist3d(T, X, "float_norm")[0] > dist3d(T, X)[0]:
                best = X
                break
        assert best is not None
        # the candidate for level l: matched while the predicted level is l (l = 0: matched only at level 1)
        add(best, sf[l], l, "ratio == sf[%d]" % l, l > 0)
        add(best, next_down(sf[l]), l, "ratio one float below sf[%d]" % l, l > 0)
        add(best, next_up(sf[l]), l, "ratio one float above sf[%d]" % l, l == 0 or l == nl - 1)
    X = _backproject(T, 320.5, 240.5, 7.0)
    add(X, F32(0.75), 0, "ratio below 1", False)
    add(X, F32(sf[-1] * F32(1.3)), nl - 1, "ratio above sf[n-1]", True)
    n = len(world)
    desc = descriptors(n)
    sc = Scene("kf-level-%s-%s" % (pose_name, scale_name), "kf", T=T, world=np.array(world, F32), scale=scale, nlevels=nl,
               cur_kps=keypoints(xy, octs), cur_desc=desc, desc=desc, min_dist=np.array(md, F32), th=th, orb_dist=TH_HIGH)
    sc.facts = facts
    return sc


def local_scene(scale_name):
    """SearchByProjection(Frame, vector<MapPoint*>): projections at (u, v) in [20, 32) with candidates at |dx| == r and one
    float beyond (r = 2.5 * th * sf[l], at a level whose powf factor differs), and a view-cosine block: cosines 0.998f (r
    2.5 in double, 4.0 against 0.998f), the float below it, 1 and 0.5, each with a candidate at 3.25 * th * sf[l]."""
    scale, nl = SCALES[scale_name]
    sf = scale_table(scale, nl)
    lev = _pow_level(scale, nl)
    th = float(F32(17.0) / F32(2.5) / sf[lev])
    proj, level, vcos, xy, octs, facts = [], [], [], [], [], []
    r = F32(F32(F32(2.5) * F32(th)) * sf[lev])
    found = 0
    for k in range(64):
        u, v = steps(F32(21.25 + 3 * k / 64), k), steps(F32(23.75 + 5 * k / 64), 3 * k)
        q = _window_queries(u, v, r)
        if q is None or found == 3:
            continue
        found += 1
        for c, lab, kept in q:
            facts.append((len(proj), lab, kept))
            proj.append((u, v)); level.append(lev); vcos.append(F32(1)); xy.append(c); octs.append(lev)
    assert len(proj) >= 16
    for c, lab, kept in ((F32(0.998), "view_cos == 0.998f: r 2.5", False), (next_down(F32(0.998)), "view_cos below 0.998f: r 4.0", True),
                         (F32(1), "view_cos 1: r 2.5", False), (F32(0.5), "view_cos 0.5: r 4.0", True)):
        u, v = F32(300.25 + 40 * len(facts) % 200), F32(200.5)
        d = F32(F32(F32(3.25) * F32(th)) * sf[lev])
        facts.append((len(proj), lab, kept))
        proj.append((u, v)); level.append(lev); vcos.append(c); xy.append((F32(u + d), v)); octs.append(lev)
    n = len(proj)
    desc = descriptors(n)
    sc = Scene("local-%s" % scale_name, "local", kps=keypoints(xy, octs), desc=desc, proj=np.array(proj, F32),
               level=np.array(level, np.int32), view_cos=np.array(vcos, F32), mp_desc=desc, th=th, nnratio=0.8, scale=scale, nlevels=nl)
    sc.facts = facts
    return sc


def compute_f12(T1, T2):
    """F12 = K^-T [t12]x R12 K^-1 of two general poses (KeyFrame-level ComputeF12), in double, rounded to float once"""
    A, B = T1.astype(F64), T2.astype(F64)
    R12 = A[:, :3] @ B[:, :3].T
    t12 = -A[:, :3] @ B[:, :3].T @ B[:, 3] + A[:, 3]
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    K = np.array([[float(FX), 0, float(CX)], [0, float(FY), float(CY)], [0, 0, 1]])
    Ki = np.linalg.inv(K)
    return (Ki.T @ tx @ R12 @ Ki).astype(F32)


def _edge_points(x1, y1, F, sig2):
    """Keypoint pairs on the epipolar decision at sigma2: (x1', y1, x2, y2) where dsqr is the largest float below
    3.84*sigma2 (kept) and where it is the first float at or above it (dropped).  num = la*x2 + lb*y2 + lc cancels, so one
    ulp of x2 moves dsqr by ~1e-5 relative; the walk moves x1 ulp by ulp (which moves den finely) and tries the x2 floats
    next to the crossing of each line.  Returns {True: (x1, y1, x2, y2), False: ...} or None."""
    thr = 3.84 * F64(F32(sig2))
    below = F32(thr)
    if F64(below) >= thr:
        below = next_down(below)
    above = next_up(below)
    Ff = F.reshape(-1)
    x1s = steps(F32(x1), np.arange(-4000, 4001))
    y1f = F32(y1)
    la, lb, lc = ((x1s * Ff[0] + y1f * Ff[3]) + Ff[6]), ((x1s * Ff[1] + y1f * Ff[4]) + Ff[7]), ((x1s * Ff[2] + y1f * Ff[5]) + Ff[8])
    den = la * la + lb * lb
    if abs(float(la[0])) < abs(float(lb[0])):   # walk the coordinate with the larger coefficient
        return None
    y2 = F32(240.0)
    x2c = (np.sqrt(thr * den.astype(F64)) - lb.astype(F64) * F64(y2) - lc.astype(F64)) / la.astype(F64)
    if not (40 < x2c[0] < 600):
        return None
    x2 = steps(x2c.astype(F32)[:, None], np.arange(-3, 4)[None, :])
    num = (la[:, None] * x2 + lb[:, None] * y2) + lc[:, None]
    dsqr = (num * num) / den[:, None]
    out = {}
    for key, target in ((True, below), (False, above)):
        hit = np.argwhere(dsqr == target)
        if not len(hit):
            return None
        i, j = hit[0]
        out[key] = (x1s[i], y1f, x2[i, j], y2)
    return out


def tri_scene(pose1, pose2, scale_name, seed):
    """SearchForTriangulation with F12 of two general poses: per side-2 level, side-1 keypoints whose only candidate sits
    where dsqr is the largest float below 3.84*sigma2 (matched) or the first float at or above it (not matched); more
    keypoints are added until every epipolar variant changes one of them."""
    scale, nl = SCALES[scale_name]
    sig2 = sigma2(scale, nl)
    F = compute_f12(POSES[pose1], POSES[pose2])
    rng = np.random.default_rng(seed)
    k1, k2, o2, facts = [], [], [], []
    need = set(VARIANTS_BY_ROUTINE["tri"])
    for l in range(nl):
        tries, placed = 0, False
        while tries < 300 and (not placed or (need and tries < 40)):
            tries += 1
            x1, y1 = F32(rng.uniform(40, 600)), F32(rng.uniform(40, 440))
            e = _edge_points(x1, y1, F, sig2[l])
            if e is None:
                continue
            got = {var for var in need for key in (True, False) if epipolar(*e[key], F, sig2[l], var)[0] != key}
            if placed and not got:
                continue
            need -= got
            placed = True
            for key in (True, False):
                facts.append((len(k1), "dsqr %s 3.84*sigma2[%d]" % ("largest float below" if key else "first float at or above", l), key))
                k1.append(e[key][:2]); k2.append(e[key][2:]); o2.append(l)
    assert not need, need
    n = len(k1)
    desc = descriptors(n)
    sc = Scene("tri-%s%s-%s" % (pose1, pose2, scale_name), "tri", k1=keypoints(k1, 0), d1=desc, k2=keypoints(k2, o2), d2=desc,
               F12=F, sig2=sig2, scale=scale, nlevels=nl)
    sc.facts = facts
    return sc


_SCENES = None


def scenes():
    global _SCENES
    if _SCENES is None:
        _SCENES = [
            bounds_scene("ff", "a", "1.2x8", 1), bounds_scene("ff", "b", "1.5x12", 2),
            bounds_scene("kf", "c", "1.2x8", 3), bounds_scene("kf", "b", "1.5x12", 4),
            window_scene("ff", "c", "1.2x8", 5), window_scene("ff", "a", "1.5x12", 6),
            window_scene("kf", "b", "1.2x8", 7), window_scene("kf", "a", "1.5x12", 8),
            window_scene("f1f2", "c", "1.2x8", 9),
            level_scene("a", "1.2x8", 10), level_scene("b", "1.5x12", 11),
            local_scene("1.2x8"), local_scene("1.5x12"),
            tri_scene("a", "b", "1.2x8", 12), tri_scene("b", "c", "1.5x12", 13),
        ]
    return _SCENES


def scene(name):
    return next(s for s in scenes() if s.name == name)


# the variants that change each scene's matches (test_oracle_projection_domain.py checks both directions)
VARIANTS = {
    'ff-bounds-a-1.2x8': ['fma_gemm', 'double_gemm', 'assoc_uv', 'fma_uv', 'bounds_inclusive'],
    'ff-bounds-b-1.5x12': ['fma_gemm', 'double_gemm', 'gemm_reversed', 'assoc_uv', 'fma_uv', 'divide_uv', 'bounds_inclusive'],
    'kf-bounds-c-1.2x8': ['fma_gemm', 'double_gemm', 'divide_uv', 'bounds_inclusive'],
    'kf-bounds-b-1.5x12': ['fma_gemm', 'double_gemm', 'assoc_uv', 'fma_uv', 'divide_uv', 'bounds_inclusive'],
    'ff-window-c-1.2x8': ['fma_gemm', 'double_gemm', 'gemm_reversed', 'assoc_uv', 'fma_uv', 'divide_uv', 'window_ge', 'radius_pow'],
    'ff-window-a-1.5x12': ['fma_gemm', 'double_gemm', 'gemm_reversed', 'assoc_uv', 'fma_uv', 'divide_uv', 'window_ge'],
    'kf-window-b-1.2x8': ['fma_gemm', 'double_gemm', 'gemm_reversed', 'assoc_uv', 'fma_uv', 'divide_uv', 'window_ge', 'radius_pow'],
    'kf-window-a-1.5x12': ['fma_gemm', 'double_gemm', 'gemm_reversed', 'assoc_uv', 'fma_uv', 'divide_uv', 'window_ge'],
    'f1f2-window-c-1.2x8': ['fma_gemm', 'double_gemm', 'gemm_reversed', 'assoc_uv', 'fma_uv', 'divide_uv', 'window_ge'],
    'kf-level-a-1.2x8': ['radius_pow', 'upper_bound', 'float_norm'],
    'kf-level-b-1.5x12': ['upper_bound', 'float_norm'],
    'local-1.2x8': ['window_ge', 'radius_pow', 'view_cos_float'],
    'local-1.5x12': ['window_ge', 'view_cos_float'],
    'tri-ab-1.2x8': ['fma_line', 'line_reordered', 'fma_num', 'float_thr'],
    'tri-bc-1.5x12': ['fma_line', 'line_reordered', 'fma_num', 'float_thr'],
}
