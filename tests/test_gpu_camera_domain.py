"""The camera half of Frame on the device, bit for bit against the oracle (every NaN equal to every NaN), which
test_oracle_camera_domain.py holds to python-cv2 and to the reference's own Frame / ORBmatcher: orbfe_undistort_keypoints,
orbfe_undistort_keypoints_device (in place and out of place) and orbfe_image_bounds on every camera model of
camera_domain_scenes.py, the half-cell grid scenes and the NaN / infinite / 2^31-overflowing windows through every windowed
entry, and one chain extract -> undistort -> bounds -> SearchByProjection on a distorted 1080p camera."""
import ctypes as C

import numpy as np
import pytest

import camera_domain_scenes as S
import oracle as O
import orb_slam_b200 as fe
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import textured_frame

pytestmark = pytest.mark.gpu

T_ID = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def same_kps(a, b):
    return all(same(a[f], b[f]) for f in ("x", "y", "size", "angle", "response")) and \
        np.array_equal(a["octave"], b["octave"]) and np.array_equal(a["class_id"], b["class_id"])


def views(kps, desc, bounds, ginv=None):
    """the library's and the oracle's view of one frame with the given bounds and grid_inv (default: Frame.cc:77-78's)"""
    gw, gh = S.grid_inv(bounds) if ginv is None else ginv
    v, o = M.FrameView(kps, desc, 64, 48), O.OracleFrame(kps, desc, 64, 48)
    for c in (v.c, o.c):
        c.min_x, c.min_y, c.max_x, c.max_y = [float(x) for x in bounds]
        c.grid_inv_w, c.grid_inv_h = float(gw), float(gh)
    O.lib().orb_oracle_frame_grid(C.byref(o.c))
    return v, o


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", 0))


# ---- undistortion and bounds -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cam", S.CAMERAS, ids=str)
def test_undistort_and_bounds(gpu_required, cam):
    pts = S.points(cam)
    n = len(pts)
    kps = S.keypoints(pts, np.arange(n) % 8, np.linspace(0, 359, n))
    want = O.undistort_keypoints(kps, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    m = fe.ORBmatcher(0.9, True)
    assert same_kps(M.undistort_keypoints(m, kps, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist), want)
    d_in, d_out = dev(kps.view(np.uint8)), dev(np.zeros(n * 28, np.uint8))
    M.undistort_keypoints_device(m, d_in.data_ptr(), d_out.data_ptr(), n, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    M.undistort_keypoints_device(m, d_in.data_ptr(), d_in.data_ptr(), n, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    m.sync()
    assert same_kps(d_out.cpu().numpy().view(S.KP_DTYPE), want)
    assert same_kps(d_in.cpu().numpy().view(S.KP_DTYPE), want)
    b = M.image_bounds(m, cam.W, cam.H, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    m.close()
    assert same(b, O.image_bounds(cam.W, cam.H, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist))
    if cam.name == "zero-den-corner":
        assert list(b[:2]) == [-2 ** 31, -2 ** 31]
    if cam.name == "k1-minus-zero":
        assert same_kps(want, kps) and list(b) == [0, 0, cam.W, cam.H]


# ---- grid scenes -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", list(S.GRID_GEOMS), ids=str)
def test_grid_scene_guided(gpu_required, geom):
    """One query per keypoint carrying its descriptor, a 0.25-px window at the keypoint and a whole-grid window:
    orbfe_guided_best (th_dist 0) finds exactly the keypoints PosInGrid keeps; orbfe_guided_search (hist 0 / 1) the same."""
    s = S.grid_scene(geom)
    v, o = views(s.kps, s.desc, s.bounds)
    n = len(s.kps)
    cx, cy = (s.bounds[0] + s.bounds[2]) / 2, (s.bounds[1] + s.bounds[3]) / 2
    qu = np.concatenate([s.kps["x"], np.full(n, cx, np.float32)])
    qv = np.concatenate([s.kps["y"], np.full(n, cy, np.float32)])
    qr = np.concatenate([np.full(n, 0.25, np.float32), np.full(n, 1e4, np.float32)])
    qd = np.concatenate([s.desc, s.desc])
    lo, hi = np.full(2 * n, -1, np.int32), np.full(2 * n, -1, np.int32)
    m = fe.ORBmatcher(0.9, False)
    best = M.guided_best(m, v, qu, qv, qr, lo, hi, qd, 0)
    assert np.array_equal(best, O.guided_best(o, qu, qv, qr, lo, hi, qd, 0))
    if geom != "min-above-max":   # with min > max every window is empty
        assert np.array_equal(best[n:] >= 0, s.cell >= 0) and (best[n:][s.cell >= 0] == np.flatnonzero(s.cell >= 0)).all()
    for hist in (0, 1):
        args = (qu, qv, qr, lo, hi, qd, np.zeros(2 * n, np.float32), 0)
        got = M.guided_search(m, v, *args, 100, hist)
        assert got[0] == O.guided_search(o, *args, 0.9, 100, hist)[0] and np.array_equal(got[1], O.guided_search(o, *args, 0.9, 100, hist)[1])
    m.close()


@pytest.mark.parametrize("geom", ["pow2-origin", "pow2-negative-min", "unit-fractional-min", "min-above-max"])
def test_grid_scene_frames_and_initialization(gpu_required, geom):
    """SearchByProjection(Frame, Frame) with the Last frame's points projecting (fx = fy = 1, cx = cy = 0) onto the Current
    keypoints, and SearchForInitialization (a grid of level-0 keypoints only) with vbPrevMatched at them."""
    s = S.grid_scene(geom)
    v, o = views(s.kps, s.desc, s.bounds)
    n = len(s.kps)
    world = np.stack([s.kps["x"], s.kps["y"], np.ones(n, np.float32)], 1).astype(np.float32)
    has, outl = np.ones(n, np.uint8), np.zeros(n, np.uint8)
    m = fe.ORBmatcher(0.9, True)
    nm, mp = M.search_by_projection_frames(m, [v], [v], [has], [outl], [world], [T_ID], 1.0, 1.0, 0.0, 0.0, 0.5)
    n_o, mp_o = O.search_by_projection_ff(o, o, has, outl, world, T_ID, 1.0, 1.0, 0.0, 0.0, 0.5)
    assert nm[0] == n_o and np.array_equal(mp[0], mp_o)
    prev = np.stack([s.kps["x"], s.kps["y"]], 1).astype(np.float32)
    n1, m12, pv = M.search_for_initialization(m, v, v, prev, 1)
    n1_o, m12_o, pv_o = O.search_for_initialization(o, o, prev, 1, nnratio=0.9)
    m.close()
    assert n1 == n1_o and np.array_equal(m12, m12_o) and same(pv, pv_o)
    if geom == "pow2-origin":
        assert n_o > 0 and n1_o > 0


# ---- windows the reference finds empty ---------------------------------------------------------------------------------------
def _win():
    s = S.window_scene()
    v, o = views(s.kps, s.desc, S.WIN_BOUNDS)
    return s, v, o


EMPTY = ["nan-u", "nan-v", "nan-uv", "nan-r", "nan-u-near-0", "nan-v-near-0", "inf-r", "inf-r-at-0", "r-at-x", "r-at-y"]


def test_window_queries_guided(gpu_required):
    """Every window of the scene alone through orbfe_guided_best and orbfe_guided_search (rule 0, hist 0 / 1): the NaN, inf-r
    and 2^31 windows are empty as in the reference (a saturating conversion scans cell 0 or the whole grid and matches), the
    controls match; then all windows in one call."""
    s, v, o = _win()
    m = fe.ORBmatcher(0.9, False)
    for q in range(s.nq):
        a = [x[q:q + 1] for x in (s.qu, s.qv, s.qr, s.qlo, s.qhi, s.qdesc)]
        b = M.guided_best(m, v, *a, 100)
        assert np.array_equal(b, O.guided_best(o, *a, 100)), s.qname[q]
        if s.qname[q] in EMPTY:
            assert b[0] == -1, s.qname[q]
        for hist in (0, 1):
            args = (*a, s.qangle[q:q + 1], 0)
            n, so = M.guided_search(m, v, *args, 100, hist)
            n_o, so_o = O.guided_search(o, *args, 0.9, 100, hist)
            assert n == n_o and np.array_equal(so, so_o), (s.qname[q], hist)
            if s.qname[q] in EMPTY:
                assert n == 0, s.qname[q]
    for name in ("whole-image", "cell-0", "r-below-x", "r-below-y"):
        assert M.guided_best(m, v, *[x[s.qname.index(name):][:1] for x in (s.qu, s.qv, s.qr, s.qlo, s.qhi, s.qdesc)], 100)[0] >= 0
    args = (s.qu, s.qv, s.qr, s.qlo, s.qhi, s.qdesc, s.qangle, 0)
    n, so = M.guided_search(m, v, *args, 100, 0)
    m.close()
    n_o, so_o = O.guided_search(o, *args, 0.9, 100, 0)
    assert n == n_o and np.array_equal(so, so_o)


@pytest.mark.parametrize("rule", [0, 1, 2])
def test_window_queries_guided_device(gpu_required, rule):
    """The same windows through orbfe_guided_search_device: one job per window and one job with all of them."""
    import torch
    s, _, o = _win()
    nq, n = s.nq, len(s.kps)
    cap = n
    kps, desc = np.tile(s.kps, (1, 1)), s.desc[None]
    qbase = np.concatenate([np.arange(nq), [0]]).astype(np.int32)
    qcnt = np.concatenate([np.ones(nq), [nq]]).astype(np.int32)
    nj = nq + 1
    Q = [dev(x) for x in (s.qu, s.qv, s.qr, s.qlo, s.qhi, s.qdesc, s.qangle)]
    d_so = dev(np.full((nj, cap), -1, np.int32))
    d_nm = torch.zeros(nj, dtype=torch.int32, device="cuda:0")
    d_k, d_d, d_c, d_f = dev(kps.view(np.uint8).reshape(1, cap, 28)), dev(desc), dev(np.array([n], np.int32)), dev(np.zeros(nj, np.int32))
    d_qb, d_qc = dev(qbase), dev(qcnt)   # held until the launch has run: a freed tensor's memory goes to the next allocation
    m = fe.ORBmatcher(0.9, False)
    M.guided_search_device(m, nj, d_k.data_ptr(), d_d.data_ptr(), d_c.data_ptr(), cap, d_f.data_ptr(), *[x.data_ptr() for x in Q],
                           d_qb.data_ptr(), d_qc.data_ptr(), nq, S.WIN_W, S.WIN_H, rule, 100, d_so.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    so, nm = d_so.cpu().numpy(), d_nm.cpu().numpy()
    for j in range(nj):
        sl = slice(int(qbase[j]), int(qbase[j] + qcnt[j]))
        n_o, so_o = O.guided_search(o, s.qu[sl], s.qv[sl], s.qr[sl], s.qlo[sl], s.qhi[sl], s.qdesc[sl], s.qangle[sl], rule, 0.9, 100, 0)
        assert nm[j] == n_o and np.array_equal(so[j], so_o), j
        if j < nq and s.qname[j] in EMPTY:
            assert nm[j] == 0, s.qname[j]


def test_window_search_f1f2_and_initialization(gpu_required):
    """WindowSearch with F1 keypoints at the NaN / infinite centres, SearchByProjection(F1, F2) with F1's map points at NaN
    and on the camera centre, SearchForInitialization with NaN / infinite vbPrevMatched (host and device forms)."""
    import torch
    s, v2, o2 = _win()
    sel = [i for i, nm in enumerate(s.qname) if not nm.startswith("r-") and nm != "nan-r" and "inf-r" not in nm]
    k1 = S.keypoints(np.stack([s.qu[sel], s.qv[sel]], 1), np.zeros(len(sel), np.int32))
    d1 = np.tile(s.base, (len(sel), 1))
    v1, o1 = views(k1, d1, S.WIN_BOUNDS)
    has = np.ones(len(sel), np.uint8)
    m = fe.ORBmatcher(1.0, False)
    n, m21 = M.window_search(m, v1, v2, has, 8)
    n_o, m21_o = O.window_search(o1, o2, has, 8, nnratio=1.0, check_orientation=False)
    assert n == n_o and np.array_equal(m21, m21_o)
    world = np.array([w for _, w in S.WORLD_SPECIAL], np.float32)
    kw = S.keypoints(np.full((len(world), 2), 5.0), np.zeros(len(world), np.int32))
    dw = np.tile(s.base, (len(world), 1))
    vw, ow = views(kw, dw, S.WIN_BOUNDS)
    valid = np.ones(len(world), np.uint8)
    n, mp = M.search_by_projection_f1f2(m, vw, v2, valid, world, T_ID, S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, 8)
    n_o, mp_o = O.search_by_projection_f1f2(ow, o2, valid, world, T_ID, S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, 8, nnratio=1.0)
    assert n == n_o and np.array_equal(mp, mp_o)
    k1["x"], k1["y"] = 5.0, 5.0
    v1, o1 = views(k1, d1, S.WIN_BOUNDS)
    prev = np.stack([s.qu[sel], s.qv[sel]], 1).astype(np.float32)
    n, m12, pv = M.search_for_initialization(m, v1, v2, prev, 8)
    n_o, m12_o, pv_o = O.search_for_initialization(o1, o2, prev, 8, nnratio=1.0, check_orientation=False)
    assert n == n_o and np.array_equal(m12, m12_o) and same(pv, pv_o)
    cap = max(len(sel), len(s.kps))
    kps = np.zeros((2, cap), S.KP_DTYPE)
    desc = np.zeros((2, cap, 32), np.uint8)
    kps[0, :len(sel)], desc[0, :len(sel)], kps[1, :len(s.kps)], desc[1, :len(s.kps)] = k1, d1, s.kps, s.desc
    pr = np.zeros((1, cap, 2), np.float32)
    pr[0, :len(sel)] = prev
    d_prev, d_m12, d_nm = dev(pr), dev(np.full((1, cap), -7, np.int32)), torch.zeros(1, dtype=torch.int32, device="cuda:0")
    d = [dev(kps.view(np.uint8).reshape(2, cap, 28)), dev(desc), dev(np.array([len(sel), len(s.kps)], np.int32)), dev(np.array([0], np.int32)),
         dev(np.array([1], np.int32))]
    M.search_for_initialization_device(m, 1, *[x.data_ptr() for x in d[:3]], cap, d[3].data_ptr(), d[4].data_ptr(), d_prev.data_ptr(),
                                       S.WIN_W, S.WIN_H, 8, d_m12.data_ptr(), d_nm.data_ptr())
    m.sync()
    m.close()
    assert int(d_nm.cpu()[0]) == n_o and np.array_equal(d_m12.cpu().numpy()[0, :len(sel)], m12_o)
    assert same(d_prev.cpu().numpy()[0, :len(sel)], pv_o)


def _sbp_device(m, s, lk, ld, world, th):
    """orbfe_search_by_projection_device: Current = the window scene, Last = (lk, ld) with `world`"""
    import torch
    n, nl = len(s.kps), len(lk)
    cap = max(n, nl)
    kps = np.zeros((2, cap), S.KP_DTYPE)
    desc = np.zeros((2, cap, 32), np.uint8)
    kps[0, :n], desc[0, :n], kps[1, :nl], desc[1, :nl] = s.kps, s.desc, lk, ld
    w = np.zeros((2, cap, 3), np.float32)
    w[1, :nl] = world
    fl = np.zeros((2, cap), np.uint8)
    fl[1, :nl] = 1
    d_mp, d_nm = dev(np.full((1, cap), -1, np.int32)), torch.zeros(1, dtype=torch.int32, device="cuda:0")
    d = [dev(kps.view(np.uint8).reshape(2, cap, 28)), dev(desc), dev(np.array([n, nl], np.int32)), dev(np.array([0], np.int32)),
         dev(np.array([1], np.int32)), dev(w), dev(fl), dev(T_ID.reshape(1, 12))]
    M.search_by_projection_device(m, 1, *[x.data_ptr() for x in d[:3]], cap, *[x.data_ptr() for x in d[3:]], S.WIN_W, S.WIN_H, 1.2, 8,
                                  S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, th, d_mp.data_ptr(), d_nm.data_ptr())
    m.sync()
    return int(d_nm.cpu()[0]), d_mp.cpu().numpy()[0, :n]


@pytest.mark.parametrize("ori", [False, True])
def test_search_by_projection_special_points(gpu_required, ori):
    """SearchByProjection(Frame, Frame) host and device forms: map points at NaN, at infinity and on the camera centre match
    nothing (as in the reference); the two control points match.  Then th one float below and at the 2^31 size for a point
    at the image centre: the whole grid, then nothing."""
    s, v, o = _win()
    n = len(S.WORLD_SPECIAL)
    lk = S.keypoints([(100.0 + 10 * i, 50.0) for i in range(n)], np.zeros(n, np.int32))
    ld = np.tile(s.base, (n, 1))
    world = np.array([w for _, w in S.WORLD_SPECIAL], np.float32)
    vl, ol = views(lk, ld, S.WIN_BOUNDS)
    has, outl = np.ones(n, np.uint8), np.zeros(n, np.uint8)
    m = fe.ORBmatcher(0.9, ori)
    nm, mp = M.search_by_projection_frames(m, [v], [vl], [has], [outl], [world], [T_ID], S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, 8.0)
    n_o, mp_o = O.search_by_projection_ff(o, ol, has, outl, world, T_ID, S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, 8.0, check_orientation=ori)
    assert nm[0] == n_o and np.array_equal(mp[0], mp_o)
    names = [x for x, _ in S.WORLD_SPECIAL]
    assert set(mp_o[mp_o >= 0].tolist()) == {names.index("centre-control")}
    nd, mpd = _sbp_device(m, s, lk, ld, world, 8.0)
    assert nd == n_o and np.array_equal(mpd, mp_o)
    c = [names.index("centre-control")]
    for th, want in ((s.r_below[0], 1), (s.r_at[0], 0)):
        nm, mp = M.search_by_projection_frames(m, [v], [views(lk[c], ld[c], S.WIN_BOUNDS)[0]], [has[c]], [outl[c]], [world[c]], [T_ID],
                                               S.WIN_FX, S.WIN_FY, S.WIN_CX, S.WIN_CY, th)
        n_o, mp_o = O.search_by_projection_ff(o, views(lk[c], ld[c], S.WIN_BOUNDS)[1], has[c], outl[c], world[c], T_ID, S.WIN_FX, S.WIN_FY,
                                              S.WIN_CX, S.WIN_CY, th, check_orientation=ori)
        assert nm[0] == n_o == want and np.array_equal(mp[0], mp_o)
        nd, mpd = _sbp_device(m, s, lk[c], ld[c], world[c], th)
        assert nd == n_o and np.array_equal(mpd, mp_o)
    m.close()


# ---- one chain on a distorted 1080p camera ---------------------------------------------------------------------------------
def test_chain_extract_undistort_bounds_sbp_1080p(gpu_required):
    """orbfe_extract_batch_device -> orbfe_undistort_keypoints_device (in place) -> orbfe_image_bounds ->
    orbfe_search_by_projection_device over 4 consecutive synthetic frames of the distorted 1080p camera, against the
    oracle's composition (extract, undistort_keypoints, image_bounds, SearchByProjection on those bounds)."""
    import torch
    cam = S.camera("hd-1080p")
    W, H, B, NF = cam.W, cam.H, 4, 1500
    base = textured_frame(W + 24, H + 24, seed=21)
    imgs = np.stack([np.ascontiguousarray(base[6 * i // 2:6 * i // 2 + H, 4 * i:4 * i + W]) for i in range(B)])
    ex = fe.ORBextractor(NF, 1.2, 8, fe.FAST_SCORE, 20, device=0)
    cap = NF
    d_img = dev(imgs)
    d_kps = torch.zeros((B, cap, 28), dtype=torch.uint8, device="cuda:0")
    d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device="cuda:0")
    d_cnt = torch.zeros(B, dtype=torch.int32, device="cuda:0")
    ex.extract_batch_device(d_img.data_ptr(), W, H, W, W * H, B, d_kps.data_ptr(), d_desc.data_ptr(), d_cnt.data_ptr())
    ex.sync()
    torch.cuda.synchronize()
    m = fe.ORBmatcher(0.9, True)
    M.undistort_keypoints_device(m, d_kps.data_ptr(), d_kps.data_ptr(), B * cap, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    b = M.image_bounds(m, W, H, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    p = O.make_params(NF, 1.2, 8, 1, 20)
    okps, odesc = [], []
    for i in range(B):
        rc, k, d, _ = O.extract(p, imgs[i])
        okps.append(O.undistort_keypoints(k, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist))
        odesc.append(d)
    ob = O.image_bounds(W, H, cam.fx, cam.fy, cam.cx, cam.cy, cam.dist)
    assert same(b, ob) and b[0] < 0 and b[2] > W
    torch.cuda.synchronize()
    cnt = d_cnt.cpu().numpy()
    kd = d_kps.cpu().numpy().view(S.KP_DTYPE).reshape(B, cap)
    for i in range(B):
        assert cnt[i] == len(okps[i]) and same_kps(kd[i, :cnt[i]], okps[i])
    # Last frame i's points: back-projected at depth 4 from its undistorted keypoints, seen by frame i + 1 after the shift
    world = np.zeros((B, cap, 3), np.float32)
    flags = np.zeros((B, cap), np.uint8)
    for i in range(B):
        k = okps[i]
        world[i, :len(k), 0] = (k["x"] - np.float32(cam.cx)) / np.float32(cam.fx) * np.float32(4)
        world[i, :len(k), 1] = (k["y"] - np.float32(cam.cy)) / np.float32(cam.fy) * np.float32(4)
        world[i, :len(k), 2] = 4
        flags[i, :len(k)] = 1
    T = np.tile(T_ID, (B - 1, 1, 1))
    T[:, 0, 3], T[:, 1, 3] = -4 * 4 / cam.fx, -3 * 4 / cam.fy
    d_mp = torch.full((B - 1, cap), -1, dtype=torch.int32, device="cuda:0")
    d_nm = torch.zeros(B - 1, dtype=torch.int32, device="cuda:0")
    # every device array is held until the launch has run: a freed tensor's memory goes to the next allocation
    d_args = [dev(np.arange(1, B, dtype=np.int32)), dev(np.arange(0, B - 1, dtype=np.int32)), dev(world), dev(flags),
              dev(T.reshape(B - 1, 12))]
    L = M._bind()
    L.orbfe_search_by_projection_device(m.handle, B - 1, C.c_void_p(d_kps.data_ptr()), C.c_void_p(d_desc.data_ptr()),
                                        C.c_void_p(d_cnt.data_ptr()), cap, *[C.c_void_p(x.data_ptr()) for x in d_args],
                                        float(b[0]), float(b[1]), float(b[2]), float(b[3]), 1.2, 8, cam.fx, cam.fy, cam.cx, cam.cy, 7.0, 1,
                                        C.c_void_p(d_mp.data_ptr()), C.c_void_p(d_nm.data_ptr()), None)
    m.sync()
    ex.close()
    m.close()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    for j in range(B - 1):
        oc = views(okps[j + 1], odesc[j + 1], ob)[1]
        ol = views(okps[j], odesc[j], ob)[1]
        nl = len(okps[j])
        n_o, mp_o = O.search_by_projection_ff(oc, ol, np.ones(nl, np.uint8), np.zeros(nl, np.uint8), world[j, :nl], T[j],
                                              cam.fx, cam.fy, cam.cx, cam.cy, 7.0, check_orientation=True)
        assert nm[j] == n_o and np.array_equal(mp[j, :len(okps[j + 1])], mp_o), j
        assert n_o > 100
