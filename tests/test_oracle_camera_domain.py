"""The camera half of Frame on the CPU: the oracle's UndistortKeyPoints / ComputeImageBounds against python-cv2 4.13's
vectors on every model of camera_domain_scenes.py (equal wherever OpenCV 2.4's loop never meets a negative denominator,
and equal to the 2.4 restatement everywhere), and the oracle's undistortion, bounds, grid, GetFeaturesInArea and
SearchByProjection(Frame, Frame) against the reference's own Frame and ORBmatcher on distorted cameras, half-cell grids and
windows with NaN, infinite and overflowing bounds."""
import ctypes as C
import os

import numpy as np
import pytest

import camera_domain_scenes as S
import oracle as O
from oracle import ref as R
from orb_slam_b200.synth import textured_frame

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "opencv_undistort_models.npz")

# points of each model on which cv2 4.13 returns something else than OpenCV 2.4's five iterations (all of them points whose
# loop meets a denominator below 0); every other model agrees on every point
SPLIT_4_13 = {"tum-fr2": 35, "div-fx200-k1-0.5": 1718, "div-fx300-k1-0.9": 1657, "div-k2-2.0": 1146, "zero-den-point": 1524,
              "zero-den-corner": 1500}


def same(a, b):
    """bit for bit, every NaN equal to every NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def needs_ref():
    if not R.available():
        pytest.skip("oracle/_ref/libref_orbslam.so not built (needs the reference sources)")


def oracle_frame(kps, desc, bounds, nlevels=8, ginv=None):
    """OracleFrame with the given image bounds and Frame.cc:77-78's grid_inv of them (or `ginv`)"""
    o = O.OracleFrame(kps, desc, 64, 48, nlevels=nlevels)
    gw, gh = S.grid_inv(bounds) if ginv is None else ginv
    o.c.min_x, o.c.min_y, o.c.max_x, o.c.max_y = [float(v) for v in bounds]
    o.c.grid_inv_w, o.c.grid_inv_h = float(gw), float(gh)
    O.lib().orb_oracle_frame_grid(C.byref(o.c))
    return o


def oracle_grid(o):
    start = np.array(o.c.cell_start, np.int32)
    return start, o.items[:start[-1]].copy()


# ---- undistortion: OpenCV 2.4 vs 4.13 ------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", S.CAMERAS, ids=str)
def test_undistortion_vs_cv2_and_the_24_loop(cam):
    g = np.load(GOLDEN)
    pts, gold = g["pts/" + cam.name], g["out/" + cam.name]
    assert np.array_equal(pts, S.points(cam))
    out = O.undistort_points(pts, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    ref24, neg = S.undistort_24(pts, cam)
    assert same(out, ref24)                                   # the oracle is 2.4's loop, on every point
    assert same(out[~neg], gold[~neg])                         # and 4.13's wherever no denominator is negative
    differ = ~np.all((out == gold) | (np.isnan(out) & np.isnan(gold)), axis=1)
    assert not np.any(differ & ~neg)
    assert int(differ.sum()) == SPLIT_4_13.get(cam.name, 0)
    if cam.name in SPLIT_4_13:   # where 4.13 exits it returns the distorted point itself (re-projected: up to rounding)
        assert np.allclose(gold[differ], pts[differ], rtol=0, atol=1e-3)
    if cam.name in S.DIVERGENT:  # the split reaches every corner ComputeImageBounds undistorts
        assert differ[:4].all()


def test_crafted_coefficients_and_points():
    """k1 = -0.0 takes Frame's `== 0` shortcut (keypoints and bounds untouched); the smallest denormal k1 does not; a
    denominator of exactly 0 gives NaN at the keypoint and, at ComputeImageBounds' (0, 0) corner, a NaN that std::min keeps
    (fminf would drop it) and Frame's int bounds turn into INT_MIN."""
    kp = S.keypoints([(10.5, 20.25), (600.0, 470.0)], [0, 3])
    c = S.camera("k1-minus-zero")
    assert np.array_equal(O.undistort_keypoints(kp, c.fx, c.fy, c.cx, c.cy, c.dist), kp)
    assert not np.array_equal(O.undistort_points(np.stack([kp["x"], kp["y"]], 1), c.fx, c.fy, c.cx, c.cy, c.dist)[:, 0], kp["x"])
    assert list(O.image_bounds(c.W, c.H, c.fx, c.fy, c.cx, c.cy, c.dist)) == [0, 0, 640, 480]
    c = S.camera("k1-denormal")
    xy = np.stack([kp["x"], kp["y"]], 1)
    assert same(np.stack([O.undistort_keypoints(kp, c.fx, c.fy, c.cx, c.cy, c.dist)[f] for f in "xy"], 1),
                O.undistort_points(xy, c.fx, c.fy, c.cx, c.cy, c.dist))
    c = S.camera("zero-den-point")
    out = O.undistort_points(np.array(c.crafted, np.float32), c.fx, c.fy, c.cx, c.cy, c.dist)
    assert np.isnan(out).all()
    c = S.camera("zero-den-corner")
    b = O.image_bounds(c.W, c.H, c.fx, c.fy, c.cx, c.cy, c.dist)
    ref24, _ = S.undistort_24(S.points(c)[:4], c)
    assert np.isnan(ref24[0]).all() and same(b, S.image_bounds_from(ref24, c))
    assert list(b) == [-2 ** 31, -2 ** 31, 6196, 253]


def test_image_bounds_every_model():
    """ComputeImageBounds = floor / ceil of the four undistorted corners through std::min / std::max (k1 == 0: the image)"""
    for c in S.CAMERAS:
        b = O.image_bounds(c.W, c.H, c.fx, c.fy, c.cx, c.cy, c.dist)
        want = S.image_bounds_from(S.undistort_24(S.points(c)[:4], c)[0], c) if c.dist[0] != 0 else [0, 0, c.W, c.H]
        assert same(b, want), c
    # the divergent cameras' bounds: min above max on both axes, or a box that crosses the image
    assert list(O.image_bounds(640, 480, 200, 200, 320, 240, S.camera("div-fx200-k1-0.5").dist)) == [640, 480, 0, 0]


# ---- the reference's own Frame -------------------------------------------------------------------------------------------
REF_CAMS = [c for c in S.CAMERAS if c.four and c.W <= 1920]


@pytest.mark.parametrize("cam", REF_CAMS, ids=str)
def test_frame_constructor_vs_reference(cam):
    """Frame(im, ..., K, DistCoef) of the reference: mvKeysUn, the image bounds, grid_inv and the grid equal the oracle's on
    every 4-coefficient model (the reference reads k1, k2, p1, p2), the divergent and zero-denominator ones included."""
    needs_ref()
    img = textured_frame(cam.W, cam.H, seed=11)
    f = R.RefFrame.from_image(img, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist[:4], 500, 1.2, 8, 1, 20)
    keys, keys_un, desc, bounds, ginv = f.get()
    start_r, items_r = f.grid()
    f.close()
    assert len(keys) > 100
    assert same(np.stack([keys_un[k] for k in "xy"], 1), np.stack([O.undistort_keypoints(keys, cam.fx, cam.fy, cam.cx, cam.cy,
                                                                                          cam.dist)[k] for k in "xy"], 1))
    b = O.image_bounds(cam.W, cam.H, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    assert same(bounds, b)
    assert same(ginv, S.frame_grid_inv(b))   # = S.grid_inv(b) unless the int difference wraps (INT_MIN bounds)
    start_o, items_o = oracle_grid(oracle_frame(keys_un, desc, b, ginv=S.frame_grid_inv(b)))
    assert np.array_equal(start_r, start_o) and np.array_equal(items_r, items_o)


@pytest.mark.parametrize("geom", list(S.GRID_GEOMS), ids=str)
def test_grid_half_cells(geom):
    """PosInGrid's round(): n + 0.5 away from zero, -0.5 dropped, -0.4 in cell 0, 63.5 / 47.5 dropped, keypoints below the
    minimum and past the maximum dropped; the oracle's grid holds exactly the designed cells.  On the origin geometry (the
    one a reference Frame of 128 x 96 has) the reference's own grid equals it."""
    s = S.grid_scene(geom)
    o = oracle_frame(s.kps, s.desc, s.bounds)
    start, items = oracle_grid(o)
    want = [[] for _ in range(64 * 48)]
    for i, c in enumerate(s.cell):
        if c >= 0:
            want[c].append(i)
    assert np.array_equal(np.diff(start), [len(w) for w in want])
    assert np.array_equal(items, [i for w in want for i in w])
    ax = np.array([a for a in S.GRID_AX for _ in S.GRID_AY])
    assert (s.cell[ax == -0.5] == -1).all() and (s.cell[ax == 63.5] == -1).all() and (s.cell[ax == 64.0] == -1).all()
    assert (s.cell[(ax == -0.4) & (s.cell >= 0)] // 48 == 0).all() and (s.cell[(ax == 62.5) & (s.cell >= 0)] // 48 == 63).all()
    if geom == "pow2-origin":
        needs_ref()
        f = R.RefFrame.from_arrays(s.kps, s.desc, 128, 96)
        start_r, items_r = f.grid()
        assert np.array_equal(start_r, start) and np.array_equal(items_r, items)
        f.close()


# ---- windows the reference finds empty -----------------------------------------------------------------------------------
def test_window_scene_is_what_it_claims():
    s = S.window_scene()
    gw, _ = S.grid_inv(S.WIN_BOUNDS)
    rb, ra = s.r_below[0], s.r_at[0]
    assert float(np.float32(np.float32(np.float32(320) + np.float32(rb)) * gw)) < 2 ** 31
    assert float(np.float32(np.float32(np.float32(320) + np.float32(ra)) * gw)) >= 2 ** 31
    assert np.nextafter(np.float32(rb), np.float32(np.inf)) == np.float32(ra)
    assert all(O.hamming(d, s.base) <= 40 for d in s.desc)
    for name, u, v, r in zip(s.qname, s.qu, s.qv, s.qr):
        rng = S.cell_range(u, v, r, S.WIN_BOUNDS)
        assert (rng is not None) == (name in ("whole-image", "cell-0", "r-below-x", "r-below-y")), name


def test_features_in_area_vs_reference():
    """GetFeaturesInArea on NaN, infinite and 2^31-overflowing windows: the reference's own Frame returns nothing (x86's
    INT_MIN conversion), the oracle equals it on every window, and the controls find keypoints."""
    needs_ref()
    s = S.window_scene()
    f = R.RefFrame.from_arrays(s.kps, s.desc, S.WIN_W, S.WIN_H)
    o = O.OracleFrame(s.kps, s.desc, S.WIN_W, S.WIN_H)
    for name, u, v, r in zip(s.qname, s.qu, s.qv, s.qr):
        for lo, hi in ((-1, -1), (0, 2), (1, 1)):
            got_r, got_o = f.features_in_area(float(u), float(v), float(r), lo, hi), o.features_in_area(float(u), float(v), float(r), lo, hi)
            assert np.array_equal(got_r, got_o), (name, lo, hi)
            if S.cell_range(u, v, r, S.WIN_BOUNDS) is None:
                assert len(got_o) == 0, name
        if name in ("whole-image", "r-below-x", "r-below-y"):
            assert len(o.features_in_area(float(u), float(v), float(r), -1, -1)) == s.kps.shape[0]
    f.close()


def sbp_last_frame(s, world_special=S.WORLD_SPECIAL):
    n = len(world_special)
    lk = S.keypoints([(100.0 + 10 * i, 50.0) for i in range(n)], np.zeros(n, np.int32))
    world = np.array([w for _, w in world_special], np.float32)
    return lk, np.tile(s.base, (n, 1)), world


T_ID = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)


@pytest.mark.parametrize("ori", [False, True])
def test_search_by_projection_frames_vs_reference(ori):
    """SearchByProjection(Frame, Frame) with map points at NaN, at infinity and on the camera centre (no depth gate, :1529-1542:
    NaN centres pass the bounds test): the reference matches only the control points, the oracle equals it."""
    needs_ref()
    s = S.window_scene()
    lk, ld, world = sbp_last_frame(s)
    has, outl = np.ones(len(lk), np.uint8), np.zeros(len(lk), np.uint8)
    fc, fl = R.RefFrame.from_arrays(s.kps, s.desc, S.WIN_W, S.WIN_H), R.RefFrame.from_arrays(lk, ld, S.WIN_W, S.WIN_H)
    n_r, mp_r = R.search_by_projection_ff(fc, fl, has, outl, world, T_ID, 8.0, check_orientation=ori)
    n_o, mp_o = O.search_by_projection_ff(O.OracleFrame(s.kps, s.desc, S.WIN_W, S.WIN_H), O.OracleFrame(lk, ld, S.WIN_W, S.WIN_H), has,
                                          outl, world, T_ID, S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, 8.0, check_orientation=ori, cur_mp=None)
    fc.close()
    fl.close()
    assert n_r == n_o and np.array_equal(mp_r, mp_o)
    names = [nm for nm, _ in S.WORLD_SPECIAL]
    assert set(mp_o[mp_o >= 0].tolist()) == {names.index("centre-control")}


def test_search_by_projection_frames_huge_radius_vs_reference():
    """th large enough that the window of a point at the image centre reaches 2^31 cells: empty in the reference; one float
    less: the whole grid."""
    needs_ref()
    s = S.window_scene()
    ws = [("centre-control", (0.0, 0.0, 3.0))]
    lk, ld, world = sbp_last_frame(s, ws)
    has, outl = np.ones(1, np.uint8), np.zeros(1, np.uint8)
    for th, matched in ((s.r_below[0], 1), (s.r_at[0], 0)):
        fc, fl = R.RefFrame.from_arrays(s.kps, s.desc, S.WIN_W, S.WIN_H), R.RefFrame.from_arrays(lk, ld, S.WIN_W, S.WIN_H)
        n_r, mp_r = R.search_by_projection_ff(fc, fl, has, outl, world, T_ID, th, check_orientation=False)
        fc.close()
        fl.close()
        n_o, mp_o = O.search_by_projection_ff(O.OracleFrame(s.kps, s.desc, S.WIN_W, S.WIN_H), O.OracleFrame(lk, ld, S.WIN_W, S.WIN_H),
                                              has, outl, world, T_ID, S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, th, check_orientation=False)
        assert n_r == n_o == matched and np.array_equal(mp_r, mp_o)


def test_window_search_and_initialization_vs_reference():
    """WindowSearch with F1 keypoints at NaN / infinite positions and SearchForInitialization with NaN / infinite
    vbPrevMatched: windows the reference finds empty; the oracle equals it."""
    needs_ref()
    s = S.window_scene()
    sel = [i for i, nm in enumerate(s.qname) if not nm.startswith("r-") and nm != "nan-r" and "inf-r" not in nm]
    f1k = S.keypoints(np.stack([s.qu[sel], s.qv[sel]], 1), np.zeros(len(sel), np.int32))
    f1d = np.tile(s.base, (len(sel), 1))
    has = np.ones(len(sel), np.uint8)
    r1, r2 = R.RefFrame.from_arrays(f1k, f1d, S.WIN_W, S.WIN_H), R.RefFrame.from_arrays(s.kps, s.desc, S.WIN_W, S.WIN_H)
    o1, o2 = O.OracleFrame(f1k, f1d, S.WIN_W, S.WIN_H), O.OracleFrame(s.kps, s.desc, S.WIN_W, S.WIN_H)
    n_r, m_r = R.window_search(r1, r2, has, 8, nnratio=1.0, check_orientation=False)
    n_o, m_o = O.window_search(o1, o2, has, 8, nnratio=1.0, check_orientation=False)
    assert n_r == n_o and np.array_equal(m_r, m_o)
    r1.close()
    f1k["x"], f1k["y"] = 5.0, 5.0          # F1 on the grid; the windows come from vbPrevMatched
    r1, o1 = R.RefFrame.from_arrays(f1k, f1d, S.WIN_W, S.WIN_H), O.OracleFrame(f1k, f1d, S.WIN_W, S.WIN_H)
    prev = np.stack([s.qu[sel], s.qv[sel]], 1).astype(np.float32)
    n_r, m_r, p_r = R.search_for_initialization(r1, r2, prev, 8, nnratio=1.0, check_orientation=False)
    n_o, m_o, p_o = O.search_for_initialization(o1, o2, prev, 8, nnratio=1.0, check_orientation=False)
    assert n_r == n_o and np.array_equal(m_r, m_o) and same(p_r, p_o)
    r1.close()
    r2.close()
