"""Camera models, points, grid scenes and window scenes for the camera half of Frame: UndistortKeyPoints and
ComputeImageBounds (reference src/Frame.cc:289-350), PosInGrid's rounding (:267-277) and GetFeaturesInArea's cell range
(:200-223).  numpy only.

- `CAMERAS`: the three cameras of golden/opencv_undistort.npz, EuRoC, TUM fr2 / fr3, a KITTI-like 1241x376 camera,
  1920x1080 and 3840x2160 cameras with fx != fy, a pure-tangential camera, three cameras on which OpenCV 2.4's five fixed
  iterations and OpenCV 4.x's early exit disagree (`DIVERGENT`), and crafted cases: k1 = -0.0 (Frame's `== 0` shortcut),
  k1 = the smallest denormal (no shortcut), and denominators of exactly 0 at a keypoint and at ComputeImageBounds' (0, 0)
  corner.
- `points(cam)`: corners, edge midpoints, sub-pixel and level-scaled positions, the crafted point, uniform points.
- `undistort_24`: a plain-Python restatement of cvUndistortPoints' loop as OpenCV 2.4 runs it (five iterations, no exit),
  which also reports whether any iteration met a denominator below 0 -- the condition on which OpenCV 4.x stops and
  returns the distorted point instead.
- `grid_scene(geom)`: keypoints at exact half-cell positions of a grid whose `grid_inv` is a power of two (n + 0.5 rounds
  away from zero, -0.5 is dropped, -0.4 lands in cell 0, 63.5 and 47.5 are dropped), below the minimum and past the
  maximum; also bounds with min > max.
- `window_scene()`: keypoints in cell (0, 0) and along the whole grid, all within Hamming distance 40 of one descriptor, and
  windows with NaN / +-inf centres, r = +-inf, NaN r and r just below and at the size where `(u - min + r) * grid_inv`
  reaches 2^31; `WORLD_SPECIAL` holds world points that project to such windows (NaN, +-inf, the camera centre).  The
  reference converts each cell bound with x86-64's float-to-int conversion: NaN, +-inf and values outside [-2^31, 2^31)
  give INT_MIN, so every such window is empty; a saturating conversion would scan cell 0 or the whole grid.
"""
import math

import numpy as np

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])
F32 = np.float32
DENORM_MIN = float(np.nextafter(F32(0), F32(1)))   # 1.4e-45, the smallest positive float
TWO31 = 2.0 ** 31


class Camera:
    def __init__(self, name, W, H, fx, fy, cx, cy, dist, crafted=None):
        self.name, self.W, self.H = name, W, H
        self.fx, self.fy, self.cx, self.cy = float(F32(fx)), float(F32(fy)), float(F32(cx)), float(F32(cy))
        d = np.zeros(5, F32)
        d[:len(dist)] = dist
        self.dist = d
        self.crafted = crafted or []   # extra (x, y) points of the model

    @property
    def four(self):
        """the reference reads k1, k2, p1, p2 (Frame's mDistCoef is 4x1): a model it can run"""
        return self.dist[4] == 0

    @property
    def K(self):
        return np.array([[self.fx, 0, self.cx], [0, self.fy, self.cy], [0, 0, 1]], np.float64)

    def __repr__(self):
        return self.name


CAMERAS = [
    # golden/opencv_undistort.npz's K with its three coefficient sets
    Camera("golden-tum-fr1", 640, 480, 517.3, 516.5, 318.6, 255.3, [0.2624, -0.9531, -0.0054, 0.0026, 1.1633]),
    Camera("golden-4coef", 640, 480, 517.3, 516.5, 318.6, 255.3, [-0.28, 0.07, 0.0002, 0.00002]),
    Camera("golden-k1", 640, 480, 517.3, 516.5, 318.6, 255.3, [0.1]),
    Camera("euroc", 752, 480, 458.654, 457.296, 367.215, 248.375, [-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05]),
    Camera("tum-fr2", 640, 480, 520.908620, 521.007327, 325.141442, 249.701764, [0.231222, -0.784899, -0.003257, -0.000105]),
    Camera("tum-fr3", 640, 480, 535.4, 539.2, 320.1, 247.6, [0.0, 0.0, 0.0, 0.0]),   # its images are undistorted: k1 = 0
    Camera("kitti-like", 1241, 376, 718.856, 718.856, 607.1928, 185.2157, [-0.3691481, 0.1968681, 0.001353473, 0.0005677587]),
    Camera("hd-1080p", 1920, 1080, 1400.0, 1390.0, 960.5, 540.25, [-0.12, 0.05, 0.001, -0.0005, -0.01]),
    Camera("uhd-4k", 3840, 2160, 2800.0, 2810.0, 1920.0, 1080.0, [-0.08, 0.02, 0.0005, 0.0003]),
    Camera("tangential", 640, 480, 500.0, 495.0, 320.0, 240.0, [1e-6, 0.0, 0.01, -0.008]),
    # 2.4 and 4.x disagree: a denominator 1 + k1 r^2 + k2 r^4 below 0 inside the image
    Camera("div-fx200-k1-0.5", 640, 480, 200.0, 200.0, 320.0, 240.0, [-0.5]),
    Camera("div-fx300-k1-0.9", 640, 480, 300.0, 300.0, 320.0, 240.0, [-0.9]),
    Camera("div-k2-2.0", 640, 480, 400.0, 400.0, 320.0, 240.0, [0.1, -2.0]),
    # crafted coefficients
    Camera("k1-minus-zero", 640, 480, 500.0, 500.0, 320.0, 240.0, [-0.0, 0.3, 0.01, 0.01]),
    Camera("k1-denormal", 640, 480, 500.0, 500.0, 320.0, 240.0, [DENORM_MIN, 0.0, 0.0, 0.0]),
    # fx a power of two: normalised (1, 1) is exact, r^2 = 2 and 1 + k1 r^2 = 0 exactly -> inf, then NaN
    Camera("zero-den-point", 640, 480, 256.0, 256.0, 320.0, 240.0, [-0.5], crafted=[(576.0, 496.0), (64.0, 240.0 - 256.0)]),
    # the same with the principal point at (fx, fy): the corner (0, 0) is normalised (-1, -1) and undistorts to NaN
    Camera("zero-den-corner", 640, 480, 256.0, 256.0, 256.0, 256.0, [-0.5]),
]
DIVERGENT = ["div-fx200-k1-0.5", "div-fx300-k1-0.9", "div-k2-2.0"]
BY_NAME = {c.name: c for c in CAMERAS}


def camera(name):
    return BY_NAME[name]


def level_scales(sf=1.2, nlevels=8):
    """ORBextractor's mvScaleFactor: a chain of float products"""
    s = [F32(1)]
    for _ in range(1, nlevels):
        s.append(F32(s[-1] * F32(sf)))
    return np.array(s, F32)


def points(cam, n_uniform=2000, seed=0):
    """(N, 2) float32: the 4 corners ComputeImageBounds undistorts, the 4 edge midpoints (they undistort outside the corner
    bounds under pincushion distortion), sub-pixel points, level-scaled positions (integer level coordinates times the
    level's scale factor, as the extractor writes them), the model's crafted points, then uniform points."""
    W, H = cam.W, cam.H
    rng = np.random.default_rng(seed)
    p = [(0, 0), (W, 0), (0, H), (W, H), (W / 2, 0), (0, H / 2), (W, H / 2), (W / 2, H)]
    p += [(0.5, 0.5), (W - 0.25, H - 0.75), (W / 2 + 0.125, H / 2 - 0.375), (cam.cx, cam.cy)]
    sc = level_scales()
    for l in range(8):
        lx, ly = rng.integers(0, int(W / sc[l]), 6), rng.integers(0, int(H / sc[l]), 6)
        p += [(float(F32(F32(a) * sc[l])), float(F32(F32(b) * sc[l]))) for a, b in zip(lx, ly)]
    p += list(cam.crafted)
    p += list(zip(rng.uniform(0, W, n_uniform), rng.uniform(0, H, n_uniform)))
    return np.array(p, np.float64).astype(F32)


def undistort_24(pts, cam):
    """cvUndistortPoints(src, dst, K, D, R = I, P = K) as OpenCV 2.4 runs it: five fixed-point iterations in double, every
    operation in OpenCV's order, no early exit.  Returns (out float32 (N, 2), negden bool (N,)): negden = an iteration met
    a denominator below 0, where OpenCV 4.x (`if (icdist < 0)`, regression_14583) returns the input point instead."""
    d = [np.float64(v) for v in cam.dist]
    k0, k1, k2, k3, k4 = d
    fx, fy, cx, cy = (np.float64(v) for v in (cam.fx, cam.fy, cam.cx, cam.cy))
    ifx, ify = np.float64(1) / fx, np.float64(1) / fy
    z = np.float64(0)
    out = np.zeros((len(pts), 2), F32)
    neg = np.zeros(len(pts), bool)
    with np.errstate(all="ignore"):
        for i, (px, py) in enumerate(np.asarray(pts, F32)):
            x = x0 = (np.float64(px) - cx) * ifx
            y = y0 = (np.float64(py) - cy) * ify
            for _ in range(5):
                r2 = x * x + y * y
                den = 1 + ((k4 * r2 + k1) * r2 + k0) * r2
                icdist = (1 + ((z * r2 + z) * r2 + z) * r2) / den
                neg[i] |= bool(icdist < 0)
                dx = 2 * k2 * x * y + k3 * (r2 + 2 * x * x)
                dy = k2 * (r2 + 2 * y * y) + 2 * k3 * x * y
                x = (x0 - dx) * icdist
                y = (y0 - dy) * icdist
            xx = fx * x + z * y + cx
            yy = z * x + fy * y + cy
            ww = np.float64(1) / (z * x + z * y + np.float64(1))
            out[i] = (F32(xx * ww), F32(yy * ww))
    return out, neg


def std_min(a, b):
    """std::min(a, b) = (b < a) ? b : a -- NaN in `a` is kept, NaN in `b` is not (fminf drops both)"""
    return b if b < a else a


def std_max(a, b):
    """std::max(a, b) = (a < b) ? b : a"""
    return b if a < b else a


def image_bounds_from(corners, cam):
    """ComputeImageBounds (:336-339) on the four undistorted corners (0,0), (W,0), (0,H), (W,H), stored in Frame's `static int`
    members (Frame.h:121-124): a NaN corner the first std::min / std::max argument keeps becomes INT_MIN"""
    c = np.asarray(corners, F32)
    f, e = np.floor, np.ceil
    b = [std_min(f(c[0, 0]), f(c[2, 0])), std_min(f(c[0, 1]), f(c[1, 1])), std_max(e(c[1, 0]), e(c[3, 0])), std_max(e(c[2, 1]), e(c[3, 1]))]
    return np.array([x86_int(v) for v in b], F32)


def grid_inv(bounds):
    """Frame.cc:77-78: FRAME_GRID_COLS / (mnMaxX - mnMinX), the difference in float (the bounds of the views here)"""
    with np.errstate(all="ignore"):
        return F32(64) / F32(bounds[2] - bounds[0]), F32(48) / F32(bounds[3] - bounds[1])


def frame_grid_inv(bounds):
    """Frame.cc:77-78 on the reference's int bounds: the difference is an int and wraps past 2^31 (INT_MIN bounds)"""
    d = [(int(bounds[2]) - int(bounds[0]) + 2 ** 31) % 2 ** 32 - 2 ** 31, (int(bounds[3]) - int(bounds[1]) + 2 ** 31) % 2 ** 32 - 2 ** 31]
    return F32(64) / F32(d[0]), F32(48) / F32(d[1])


def x86_int(v):
    """(int) of a float or double as x86-64's cvttss2si / cvttsd2si: truncation, INT_MIN for NaN and outside [-2^31, 2^31)"""
    v = float(v)
    if not (-TWO31 <= v < TWO31):
        return -2 ** 31
    return int(v)


def cell_range(u, v, r, bounds):
    """GetFeaturesInArea's cell range (Frame.cc:205-223) in float arithmetic, or None when the window is empty"""
    gw, gh = grid_inv(bounds)
    with np.errstate(all="ignore"):
        u, v, r = F32(u), F32(v), F32(r)
        x0 = max(0, x86_int(np.floor((u - F32(bounds[0]) - r) * gw)))
        if x0 >= 64:
            return None
        x1 = min(63, x86_int(np.ceil((u - F32(bounds[0]) + r) * gw)))
        if x1 < 0:
            return None
        y0 = max(0, x86_int(np.floor((v - F32(bounds[1]) - r) * gh)))
        if y0 >= 48:
            return None
        y1 = min(47, x86_int(np.ceil((v - F32(bounds[1]) + r) * gh)))
        if y1 < 0:
            return None
    return x0, x1, y0, y1


def _desc_near(base, k, rng):
    """base with k distinct bits flipped"""
    d = base.copy()
    for b in rng.choice(256, k, replace=False):
        d[b // 8] ^= np.uint8(1 << (b % 8))
    return d


def random_desc(n, rng):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


def keypoints(xy, octaves, angles=None):
    k = np.zeros(len(xy), KP_DTYPE)
    if len(xy):
        xy = np.asarray(xy, F32)
        k["x"], k["y"] = xy[:, 0], xy[:, 1]
    k["octave"] = octaves
    k["angle"] = 0.0 if angles is None else angles
    k["size"], k["response"], k["class_id"] = 31.0, 1.0, -1
    return k


# ---- grid scenes -------------------------------------------------------------------------------------------------------
# (min_x, min_y, max_x, max_y): grid_inv 0.5 / 0.5, 0.5 / 0.5 with negative minima, 1 / 1 with fractional minima, -0.5 / -0.5
GRID_GEOMS = {
    "pow2-origin": (0.0, 0.0, 128.0, 96.0),
    "pow2-negative-min": (-16.0, -8.0, 112.0, 88.0),
    "unit-fractional-min": (-37.25, -20.5, 26.75, 27.5),
    "min-above-max": (130.0, 100.0, 2.0, 4.0),
}
# grid coordinates (x - min) * grid_inv of the keypoints; each is exact in float for the geometries above
GRID_AX = [-1.0, -0.5, -0.4, 0.0, 0.4, 0.5, 1.5, 2.5, 31.5, 62.4, 62.5, 63.0, 63.4, 63.5, 64.0, 70.0]
GRID_AY = [-0.5, -0.4, 0.0, 0.5, 23.5, 46.5, 47.4, 47.5, 50.0]


class GridScene:
    pass


def grid_scene(name, seed=3):
    """Keypoints at every (GRID_AX, GRID_AY) grid coordinate of geometry `name`, octaves cycling over 0..7 (every sixth one
    at level 0 for SearchForInitialization's grid), distinct random descriptors; `cell[i]` = PosInGrid's cell or -1."""
    b = GRID_GEOMS[name]
    gw, gh = grid_inv(b)
    xy, cells = [], []
    for ax in GRID_AX:
        for ay in GRID_AY:
            x, y = F32(F32(b[0]) + F32(ax) / gw), F32(F32(b[1]) + F32(ay) / gh)
            gx, gy = float(F32((x - F32(b[0])) * gw)), float(F32((y - F32(b[1])) * gh))
            if ax * 2 == int(ax * 2) and ay * 2 == int(ay * 2):   # the half-cell and whole-cell coordinates are exact
                assert gx == ax and gy == ay
            xy.append((x, y))
            px, py = x86_int(_round_half_away(gx)), x86_int(_round_half_away(gy))
            cells.append(px * 48 + py if 0 <= px < 64 and 0 <= py < 48 else -1)
    n = len(xy)
    rng = np.random.default_rng(seed)
    s = GridScene()
    s.name, s.bounds, s.gw, s.gh = name, b, gw, gh
    s.kps = keypoints(xy, np.arange(n) % 6 % 8)
    s.desc = random_desc(n, rng)
    s.cell = np.array(cells, np.int32)
    return s


def _round_half_away(a):
    return math.copysign(math.floor(abs(a) + 0.5), a)


# ---- window scenes -----------------------------------------------------------------------------------------------------
WIN_W, WIN_H = 640, 480
WIN_BOUNDS = (0.0, 0.0, float(WIN_W), float(WIN_H))
WIN_FX = WIN_FY = 500.0
WIN_CX, WIN_CY = 320.0, 240.0


def overflow_radius(u, lo, ginv):
    """(r_below, r_at): the largest float r with (u - lo + r) * ginv below 2^31 in float arithmetic, and the next float"""
    u, lo, ginv = F32(u), F32(lo), F32(ginv)
    f = lambda r: float(F32(F32(F32(u - lo) + F32(r)) * ginv))
    r = F32(TWO31 / float(ginv))
    while f(r) >= TWO31:
        r = np.nextafter(r, F32(0))
    while f(np.nextafter(r, F32(np.inf))) < TWO31:
        r = np.nextafter(r, F32(np.inf))
    return float(r), float(np.nextafter(r, F32(np.inf)))


class WindowScene:
    pass


def window_scene(seed=5):
    """Keypoints at every octave in cell (0, 0) and one in every 7th cell of the grid, all within Hamming distance 40 of
    `base`, so that any keypoint a window reaches is matched by a query carrying `base`.  Queries (u, v, r) with names."""
    rng = np.random.default_rng(seed)
    gw, gh = grid_inv(WIN_BOUNDS)
    xy, oct_ = [], []
    for o in range(8):                        # cell (0, 0) at every octave, the cells next to it, and the image centre
        xy += [(0.5 + 0.125 * o, 0.25 + 0.125 * o), (3.0 + 0.25 * o, 2.0), (14.0, 1.0 + o), (321.0 - 0.5 * o, 241.0 - 0.25 * o)]
        oct_ += [o, o, o, o]
    for c in range(0, 64 * 48, 7):            # along the whole grid
        ix, iy = divmod(c, 48)
        xy.append((float(F32(ix) / gw) + 0.25, float(F32(iy) / gh) + 0.5))
        oct_.append(c % 3)
    n = len(xy)
    s = WindowScene()
    s.base = random_desc(1, rng)[0]
    s.kps = keypoints(xy, np.array(oct_, np.int32), rng.uniform(0, 360, n))
    s.desc = np.stack([_desc_near(s.base, int(rng.integers(1, 40)), rng) for _ in range(n)])
    inf, nan = math.inf, math.nan
    rb_x, ra_x = overflow_radius(320.0, 0.0, gw)
    rb_y, ra_y = overflow_radius(240.0, 0.0, gh)
    q = [  # (name, u, v, r): r_at* make (u - min + r) * grid_inv reach 2^31, r_below* stay one float below
        ("nan-u", nan, 240.0, 8.0), ("nan-v", 320.0, nan, 8.0), ("nan-uv", nan, nan, 8.0), ("nan-r", 320.0, 240.0, nan),
        ("nan-u-near-0", nan, 2.0, 8.0), ("nan-v-near-0", 2.0, nan, 8.0),
        ("inf-u", inf, 240.0, 8.0), ("minus-inf-u", -inf, 240.0, 8.0), ("inf-v", 320.0, inf, 8.0), ("minus-inf-v", 2.0, -inf, 8.0),
        ("inf-r", 320.0, 240.0, inf), ("minus-inf-r", 320.0, 240.0, -inf), ("inf-r-at-0", 0.0, 0.0, inf),
        ("r-below-x", 320.0, 240.0, rb_x), ("r-at-x", 320.0, 240.0, ra_x),
        ("r-below-y", 320.0, 240.0, rb_y), ("r-at-y", 320.0, 240.0, ra_y),
        ("huge-u", 3e10, 240.0, 0.0), ("huge-negative-u", -3e10, 240.0, 8.0),
        ("whole-image", 320.0, 240.0, 1000.0), ("cell-0", 1.0, 1.0, 4.0),   # controls: windows both sides scan
    ]
    s.qname = [x[0] for x in q]
    s.qu = np.array([x[1] for x in q], F32)
    s.qv = np.array([x[2] for x in q], F32)
    s.qr = np.array([x[3] for x in q], F32)
    s.nq = len(q)
    s.qdesc = np.tile(s.base, (s.nq, 1))
    s.qangle = np.zeros(s.nq, F32)
    s.qlo = np.full(s.nq, -1, np.int32)
    s.qhi = np.full(s.nq, -1, np.int32)
    s.r_at = (ra_x, ra_y)
    s.r_below = (rb_x, rb_y)
    return s


# world points for SearchByProjection(Frame, Frame) under the identity pose with WIN_FX, WIN_CX: each projects to a window
# the reference finds empty (a NaN centre, or an infinite one rejected by the bounds test) but the control, at the centre
WORLD_SPECIAL = [
    ("camera-centre", (0.0, 0.0, 0.0)),              # invzc = inf, u = 0 * inf = NaN
    ("nan", (math.nan, math.nan, math.nan)),
    ("nan-x", (math.nan, 0.1, 2.0)),                  # u NaN, v finite
    ("behind-centre", (0.0, 0.0, -0.0)),             # invzc = -inf
    ("inf-all", (math.inf, math.inf, math.inf)),      # invzc = 0, u = inf * 0 = NaN
    ("inf-x", (math.inf, 0.0, 1.0)),                  # u = inf: rejected by u > mnMaxX
    ("inf-z", (1.0, 1.0, math.inf)),                  # Rcw * x3Dw adds 0 * inf: xc = yc = NaN
    ("on-axis-y", (0.0, 1.0, 0.0)),                   # u NaN, v = inf: rejected by v
    ("centre-control", (0.0, 0.0, 3.0)),              # u = cx, v = cy
]
