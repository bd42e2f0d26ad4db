"""The camera-table matchers (orbfe_search_by_projection_cams_device, orbfe_search_for_initialization_cams_device,
orbfe_guided_search_cams_device) on a three-camera rig extracted in one orbfe_extract_multi_device call: 1920 x 1080,
1280 x 720 and a distorted 1280 x 720 camera whose bounds come from orbfe_image_bounds, three frames each.

Every pair or job of one camera-table launch equals the single-geometry entry called with that pair's camera and the
oracle, output for output: SearchByProjection(Frame, Frame) with the histogram on and off and with the candidate entries
in the global scratch; cross-camera SearchForInitialization including vbPrevMatched; the guided search under rules 0-2
with occupied slots.  Then pair order, shared frames, an unused camera, eight geometries in one table, a bad camera index
(alone and beside a scratch overflow) and the matcher's stream-order rule."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle as O
import orb_slam_b200 as fe
import projection_domain_scenes as PS
from orb_slam_b200 import matching as M
from orb_slam_b200.synth import textured_frame

pytestmark = pytest.mark.gpu

F32 = np.float32
PARAMS = (1000, 1.2, 8, fe.FAST_SCORE, 20)
B = 3                        # frames per camera
TH = 7.0                     # SearchByProjection's th
DIST = (-0.28, 0.09, 0.0012, -0.0008, 0.0)
SPIN = 100_000_000           # torch.cuda._sleep cycles: one bounded spin of roughly 50 ms on an H100
# (W, H, dist, crop origin in the shared base texture): the two 720p cameras see different parts of the scene, the
# 1080p camera's top-left corner is what the undistorted 720p camera sees
CAMERAS = [(1920, 1080, None, (0, 0)), (1280, 720, None, (0, 0)), (1280, 720, DIST, (200, 300))]


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def dev(a):
    torch, d = _torch()
    return torch.from_numpy(np.ascontiguousarray(a)).to(d)


def vp(x):
    return C.c_void_p(x.data_ptr())


class Rig:
    """The rig's frame store on the device, its host copy, the camera table and the frame-camera array"""

    def __init__(self):
        torch, d = _torch()
        base = textured_frame(1920 + 3 * B + 320, 1080 + 2 * B + 220, seed=61)
        groups, self.frames = [], []
        for W, H, _, (ox, oy) in CAMERAS:
            fr = np.stack([np.ascontiguousarray(base[oy + 2 * i:oy + 2 * i + H, ox + 3 * i:ox + 3 * i + W]) for i in range(B)])
            self.frames.append(fr)
            groups.append(torch.from_numpy(fr).to(d))
        ex = fe.ORBextractor(*PARAMS)
        m = fe.ORBmatcher(0.9, True)
        try:
            self.cap = int(ex.tables()[2].sum())
            self.F = B * len(CAMERAS)
            self.kps = torch.zeros((self.F, self.cap, 28), dtype=torch.uint8, device=d)
            self.desc = torch.zeros((self.F, self.cap, 32), dtype=torch.uint8, device=d)
            self.cnt = torch.full((self.F,), -1, dtype=torch.int32, device=d)
            ex.extract_multi_device([(g.data_ptr(), W, H, W, W * H, B) for g, (W, H, _, _) in zip(groups, CAMERAS)],
                                    self.kps.data_ptr(), self.desc.data_ptr(), self.cnt.data_ptr())
            torch.cuda.synchronize()
            self.cams = []
            for W, H, dist, _ in CAMERAS:
                fx, cx, cy = F32(0.7 * W), F32(W / 2 + 0.5), F32(H / 2 - 0.5)
                b = M.image_bounds(m, W, H, fx, fx, cx, cy, dist) if dist else np.array([0, 0, W, H], F32)
                self.cams.append(tuple(float(v) for v in b) + (float(fx), float(fx), float(cx), float(cy)))
        finally:
            ex.close()
            m.close()
        assert self.cams[2][0] < 0 and self.cams[2][2] > 1280, self.cams[2]   # barrel distortion widens the bounds
        self.frame_cam = np.repeat(np.arange(len(CAMERAS), dtype=np.int32), B)
        self.d_frame_cam = dev(self.frame_cam)
        self.h_kps = self.kps.cpu().numpy().view(fe.KP_DTYPE).reshape(self.F, self.cap)
        self.h_desc = self.desc.cpu().numpy()
        self.h_cnt = self.cnt.cpu().numpy()
        assert (self.h_cnt > 500).all(), self.h_cnt
        # map point of every feature: its keypoint back-projected at depth 4 through its frame's camera
        self.world = np.zeros((self.F, self.cap, 3), F32)
        self.flags = np.zeros((self.F, self.cap), np.uint8)
        for f in range(self.F):
            n, (_, _, _, _, fx, fy, cx, cy) = self.h_cnt[f], self.cams[self.frame_cam[f]]
            k = self.h_kps[f, :n]
            self.world[f, :n, 0] = (k["x"] - F32(cx)) / F32(fx) * F32(4)
            self.world[f, :n, 1] = (k["y"] - F32(cy)) / F32(fy) * F32(4)
            self.world[f, :n, 2] = 4
            self.flags[f, :n] = 1
        self.d_world, self.d_flags = dev(self.world), dev(self.flags)

    def store(self):
        return [vp(self.kps), vp(self.desc), vp(self.cnt)]

    def oframe(self, f, cam=None):
        """the oracle's Frame of frame f with the bounds and grid of camera `cam` (default: the frame's own)"""
        n = self.h_cnt[f]
        o = O.OracleFrame(self.h_kps[f, :n], self.h_desc[f, :n], 64, 48)
        x0, y0, x1, y1 = self.cams[self.frame_cam[f] if cam is None else cam][:4]
        o.c.min_x, o.c.min_y, o.c.max_x, o.c.max_y = x0, y0, x1, y1
        o.c.grid_inv_w, o.c.grid_inv_h = float(F32(64) / F32(F32(x1) - F32(x0))), float(F32(48) / F32(F32(y1) - F32(y0)))
        O.lib().orb_oracle_frame_grid(C.byref(o.c))
        return o


@functools.lru_cache(maxsize=None)
def rig():
    return Rig()


def counters(m):
    return m.counters()[2]


def sync_error(m):
    try:
        m.sync()
        return None
    except fe.OrbfeError as e:
        return e


# ---------------------------------------------------------------------------------------------------------------------
# SearchByProjection(Frame, Frame)
# ---------------------------------------------------------------------------------------------------------------------
def sbp_pairs():
    """per camera (1, 0), (2, 1) and (2, 0): the last two share their Current frame, the first and last their Last frame"""
    return [(f0 + a, f0 + b) for f0 in (0, B, 2 * B) for a, b in ((1, 0), (2, 1), (2, 0))]


def poses(pairs):
    T = []
    for j, (c, l) in enumerate(pairs):
        fx, fy = rig().cams[rig().frame_cam[c]][4:6]
        s = (c - l) % B or B
        T.append(PS.pose((0.2, 0.3 * (-1) ** j, 0.93), 0.02 + 0.01 * (j % 3), (-3 * s * 4 / fx, -2 * s * 4 / fy, 0.01)))
    return np.stack(T).astype(F32).reshape(len(pairs), 12)


def sbp_cams(pairs, T, ori=True, cams=None, frame_cam=None, mp0=None):
    """one camera-table call: (cur_mp rows, nmatches, sync error, launches it added)"""
    torch, d = _torch()
    R = rig()
    P = len(pairs)
    d_mp = dev(np.full((P, R.cap), -1, np.int32) if mp0 is None else mp0)
    d_nm = torch.full((P,), -9, dtype=torch.int32, device=d)
    d_cur, d_last, d_T = dev(np.array([c for c, _ in pairs], np.int32)), dev(np.array([l for _, l in pairs], np.int32)), dev(T)
    m = fe.ORBmatcher(0.9, ori)
    try:
        n0 = counters(m)
        M.search_by_projection_cams_device(m, P, *[x.value for x in R.store()], R.cap, d_cur.data_ptr(), d_last.data_ptr(),
                                           R.d_world.data_ptr(), R.d_flags.data_ptr(), d_T.data_ptr(), R.cams if cams is None else cams,
                                           (R.d_frame_cam if frame_cam is None else frame_cam).data_ptr(), 1.2, 8, TH,
                                           d_mp.data_ptr(), d_nm.data_ptr())
        added = counters(m) - n0
        err = sync_error(m)
        return d_mp.cpu().numpy(), d_nm.cpu().numpy(), err, added
    finally:
        m.close()


def sbp_single(pairs, T, cam, ori=True, mp0=None):
    """the single-geometry entry on `pairs` with camera `cam` (a table row)"""
    torch, d = _torch()
    R = rig()
    P = len(pairs)
    d_mp = dev(np.full((P, R.cap), -1, np.int32) if mp0 is None else mp0)
    d_nm = torch.full((P,), -9, dtype=torch.int32, device=d)
    d_cur, d_last, d_T = dev(np.array([c for c, _ in pairs], np.int32)), dev(np.array([l for _, l in pairs], np.int32)), dev(T)
    m = fe.ORBmatcher(0.9, ori)
    try:
        x0, y0, x1, y1, fx, fy, cx, cy = cam
        rc = M._bind().orbfe_search_by_projection_device(
            m.handle, P, *R.store(), R.cap, vp(d_cur), vp(d_last), vp(R.d_world), vp(R.d_flags), vp(d_T), x0, y0, x1, y1, 1.2, 8,
            fx, fy, cx, cy, TH, int(ori), vp(d_mp), vp(d_nm), None)
        assert rc == 0
        m.sync()
        return d_mp.cpu().numpy(), d_nm.cpu().numpy()
    finally:
        m.close()


def sbp_want(pairs, T, ori=True, cam_of=None, mp0=None):
    """per pair the single-geometry entry's (row, nmatches), each camera's pairs in one call; cam_of(cur) = table row"""
    R = rig()
    cam_of = cam_of or (lambda f: R.cams[R.frame_cam[f]])
    mp, nm = np.zeros((len(pairs), R.cap), np.int32), np.zeros(len(pairs), np.int32)
    for cam in {cam_of(c) for c, _ in pairs}:
        js = [j for j, (c, _) in enumerate(pairs) if cam_of(c) == cam]
        sub = None if mp0 is None else mp0[js]
        mp[js], nm[js] = sbp_single([pairs[j] for j in js], T[js], cam, ori, sub)
    return mp, nm


def sbp_oracle(pairs, T, ori):
    R = rig()
    out = []
    for j, (c, l) in enumerate(pairs):
        nl = R.h_cnt[l]
        _, _, _, _, fx, fy, cx, cy = R.cams[R.frame_cam[c]]
        out.append(O.search_by_projection_ff(R.oframe(c), R.oframe(l), np.ones(nl, np.uint8), np.zeros(nl, np.uint8), R.world[l, :nl],
                                             T[j].reshape(3, 4), fx, fy, cx, cy, TH, check_orientation=ori))
    return out


@pytest.mark.parametrize("scratch", [False, True], ids=["smem", "scratch"])
@pytest.mark.parametrize("ori", [True, False], ids=["hist", "nohist"])
def test_projection_search_over_the_rig_in_one_launch(gpu_required, monkeypatch, ori, scratch):
    if scratch:
        monkeypatch.setenv("ORBFE_SBP_FORCE_SCRATCH", "1")
    R = rig()
    pairs = sbp_pairs()
    T = poses(pairs)
    mp, nm, err, added = sbp_cams(pairs, T, ori)
    assert err is None and added == 1
    want_mp, want_nm = sbp_want(pairs, T, ori)
    assert np.array_equal(nm, want_nm) and np.array_equal(mp, want_mp)
    for j, (n_o, mp_o) in enumerate(sbp_oracle(pairs, T, ori)):
        c = pairs[j][0]
        assert nm[j] == n_o and np.array_equal(mp[j, :R.h_cnt[c]], mp_o), pairs[j]
    assert all(nm[j] > 50 for j, (c, l) in enumerate(pairs) if c - l == 1), nm


def test_projection_search_with_occupied_slots(gpu_required):
    R = rig()
    pairs = sbp_pairs()
    T = poses(pairs)
    mp0 = np.full((len(pairs), R.cap), -1, np.int32)
    mp0[:, ::5] = 7
    mp, nm, err, _ = sbp_cams(pairs, T, mp0=mp0)
    assert err is None
    want_mp, want_nm = sbp_want(pairs, T, mp0=mp0)
    assert np.array_equal(nm, want_nm) and np.array_equal(mp, want_mp)


# ---------------------------------------------------------------------------------------------------------------------
# SearchForInitialization across cameras
# ---------------------------------------------------------------------------------------------------------------------
def init_run(pairs, prev, cams_call, cam=None, ori=True):
    """(match12 rows, nmatches, prev_matched rows) of one call: the camera-table entry, or the single-geometry entry with
    the bounds of table row `cam`"""
    torch, d = _torch()
    R = rig()
    P = len(pairs)
    d_prev, d_m12 = dev(prev), dev(np.full((P, R.cap), -5, np.int32))
    d_nm = torch.full((P,), -9, dtype=torch.int32, device=d)
    d_f1, d_f2 = dev(np.array([a for a, _ in pairs], np.int32)), dev(np.array([b for _, b in pairs], np.int32))
    m = fe.ORBmatcher(0.9, ori)
    try:
        n0 = counters(m)
        if cams_call:
            M.search_for_initialization_cams_device(m, P, *[x.value for x in R.store()], R.cap, d_f1.data_ptr(), d_f2.data_ptr(),
                                                    d_prev.data_ptr(), R.cams, R.d_frame_cam.data_ptr(), 100, d_m12.data_ptr(),
                                                    d_nm.data_ptr())
            assert counters(m) - n0 == 1
        else:
            x0, y0, x1, y1 = cam[:4]
            rc = M._bind().orbfe_search_for_initialization_device(m.handle, P, *R.store(), R.cap, vp(d_f1), vp(d_f2), vp(d_prev),
                                                                  x0, y0, x1, y1, 100, 0.9, int(ori), vp(d_m12), vp(d_nm), None)
            assert rc == 0
        m.sync()
        return d_m12.cpu().numpy(), d_nm.cpu().numpy(), d_prev.cpu().numpy()
    finally:
        m.close()


@pytest.mark.parametrize("ori", [True, False], ids=["hist", "nohist"])
def test_cross_camera_initialization_in_one_launch(gpu_required, ori):
    """F1 720p -> F2 1080p and the reverse (the 720p camera sees the 1080p camera's top-left corner), the distorted camera
    against both, and same-camera pairs, window 100, vbPrevMatched = F1's keypoints"""
    R = rig()
    pairs = [(3, 0), (0, 3), (4, 1), (1, 5), (6, 7), (7, 0), (2, 8), (3, 4), (0, 1)]
    prev = np.zeros((len(pairs), R.cap, 2), F32)
    for j, (f1, _) in enumerate(pairs):
        n = R.h_cnt[f1]
        prev[j, :n, 0], prev[j, :n, 1] = R.h_kps[f1, :n]["x"], R.h_kps[f1, :n]["y"]
    m12, nm, pm = init_run(pairs, prev, True, ori=ori)
    for cam in set(R.frame_cam[[b for _, b in pairs]]):
        js = [j for j, (_, f2) in enumerate(pairs) if R.frame_cam[f2] == cam]
        w12, wnm, wpm = init_run([pairs[j] for j in js], prev[js], False, R.cams[cam], ori)
        assert np.array_equal(nm[js], wnm) and np.array_equal(m12[js], w12), cam
        assert np.array_equal(pm[js].view(np.uint32), wpm.view(np.uint32)), cam
    for j, (f1, f2) in enumerate(pairs):
        n1 = R.h_cnt[f1]
        n_o, m12_o, prev_o = O.search_for_initialization(R.oframe(f1), R.oframe(f2), prev[j, :n1], 100, nnratio=0.9,
                                                         check_orientation=ori)
        assert nm[j] == n_o and np.array_equal(m12[j, :n1], m12_o), (f1, f2)
        assert np.array_equal(pm[j, :n1].view(np.uint32), prev_o.view(np.uint32)), (f1, f2)
    assert nm[0] > 50 and nm[1] > 50, nm   # the cross-camera pairs over a shared view match


# ---------------------------------------------------------------------------------------------------------------------
# guided search
# ---------------------------------------------------------------------------------------------------------------------
class Jobs:
    """one job per frame (searched frame f, queries = the features of the camera's previous frame moved by the 3, 2 px
    shift, windows of 8 px times the level's scale; every other query without octave filter) and a few jobs on shared
    frames; slots occupied on entry every 6th feature"""

    def __init__(self):
        R = rig()
        self.frames = list(range(R.F)) + [4, 7, 0]
        qu, qv, qr, qlo, qhi, qd, qa, base, cnt = [], [], [], [], [], [], [], [], []
        n0 = 0
        for j, f in enumerate(self.frames):
            src = f - 1 if f % B else f + 1
            k, dsc = R.h_kps[src, :R.h_cnt[src]], R.h_desc[src, :R.h_cnt[src]]
            step = 1 if j < R.F else 2
            k, dsc = k[::step], dsc[::step]
            sh = -1 if f > src else 1   # frame i shows the scene moved by (-3i, -2i)
            qu.append(k["x"] + F32(3 * sh))
            qv.append(k["y"] + F32(2 * sh))
            qr.append(F32(8) * F32(1.2) ** k["octave"].astype(F32))
            lo = np.where(np.arange(len(k)) % 2 == 0, k["octave"] - 1, -1).astype(np.int32)
            qlo.append(lo)
            qhi.append(np.where(lo == -1, -1, k["octave"] + 1).astype(np.int32))
            qd.append(dsc)
            qa.append(k["angle"])
            base.append(n0)
            cnt.append(len(k))
            n0 += len(k)
        cat = lambda xs, t: np.ascontiguousarray(np.concatenate(xs), t)
        self.h = dict(qu=cat(qu, F32), qv=cat(qv, F32), qr=cat(qr, F32), qlo=cat(qlo, np.int32), qhi=cat(qhi, np.int32),
                      qdesc=cat(qd, np.uint8), qangle=cat(qa, F32))
        self.base, self.cnt = np.array(base, np.int32), np.array(cnt, np.int32)
        self.qcap = int(self.cnt.max())
        self.d = [dev(self.h[n]) for n in ("qu", "qv", "qr", "qlo", "qhi", "qdesc", "qangle")]
        self.owner0 = np.full((len(self.frames), R.cap), -1, np.int32)
        self.owner0[:, 3::6] = 90000

    def run(self, js, rule, ori, cam=None):
        """jobs js in one call: the camera-table entry (cam None) or the single-geometry entry with table row `cam`"""
        torch, d = _torch()
        R = rig()
        n = len(js)
        d_so, d_nm = dev(self.owner0[js]), torch.full((n,), -9, dtype=torch.int32, device=d)
        d_fi, d_b, d_c = dev(np.array(self.frames, np.int32)[js]), dev(self.base[js]), dev(self.cnt[js])
        th = 50 if rule == 0 else 100
        m = fe.ORBmatcher(0.8, ori)
        try:
            if cam is None:
                M.guided_search_cams_device(m, n, *[x.value for x in R.store()], R.cap, d_fi.data_ptr(), *[x.data_ptr() for x in self.d],
                                            d_b.data_ptr(), d_c.data_ptr(), self.qcap, R.cams, R.d_frame_cam.data_ptr(), rule, th,
                                            d_so.data_ptr(), d_nm.data_ptr())
            else:
                x0, y0, x1, y1 = cam[:4]
                rc = M._bind().orbfe_guided_search_device(m.handle, n, *R.store(), R.cap, vp(d_fi), *[vp(x) for x in self.d], vp(d_b),
                                                          vp(d_c), self.qcap, x0, y0, x1, y1, rule, F32(0.8), th, int(ori), vp(d_so),
                                                          vp(d_nm), None)
                assert rc == 0
            m.sync()
            return d_so.cpu().numpy(), d_nm.cpu().numpy()
        finally:
            m.close()


@functools.lru_cache(maxsize=None)
def jobs():
    return Jobs()


@pytest.mark.parametrize("ori", [True, False], ids=["hist", "nohist"])
@pytest.mark.parametrize("rule", [0, 1, 2])
def test_guided_search_over_the_rig_in_one_launch(gpu_required, rule, ori):
    R, J = rig(), jobs()
    every = list(range(len(J.frames)))
    so, nm = J.run(every, rule, ori)
    for cam in range(len(CAMERAS)):
        js = [j for j in every if R.frame_cam[J.frames[j]] == cam]
        wso, wnm = J.run(js, rule, ori, R.cams[cam])
        assert np.array_equal(nm[js], wnm) and np.array_equal(so[js], wso), cam
    th = 50 if rule == 0 else 100
    for j, f in enumerate(J.frames):
        s = slice(J.base[j], J.base[j] + J.cnt[j])
        h = J.h
        n_o, so_o = O.guided_search(R.oframe(f), h["qu"][s], h["qv"][s], h["qr"][s], h["qlo"][s], h["qhi"][s], h["qdesc"][s],
                                    h["qangle"][s], rule, F32(0.8), th, int(ori), J.owner0[j, :R.h_cnt[f]])
        assert nm[j] == n_o and np.array_equal(so[j, :R.h_cnt[f]], so_o), (rule, f)
        assert (so[j, R.h_cnt[f]:] == J.owner0[j, R.h_cnt[f]:]).all()
    assert (nm[:R.F] > 50).all(), nm


# ---------------------------------------------------------------------------------------------------------------------
# pair order, shared frames, table layout
# ---------------------------------------------------------------------------------------------------------------------
def test_pair_order_and_table_layout_do_not_change_results(gpu_required):
    """the pairs shuffled and interleaved across cameras; then the table permuted with a fourth camera no pair uses and
    the frame cameras remapped"""
    torch, d = _torch()
    R = rig()
    pairs = sbp_pairs()
    T = poses(pairs)
    mp, nm, err, _ = sbp_cams(pairs, T)
    assert err is None
    for seed in (1, 2):
        order = np.random.default_rng(seed).permutation(len(pairs))
        smp, snm, err, _ = sbp_cams([pairs[j] for j in order], T[order])
        assert err is None and np.array_equal(snm, nm[order]) and np.array_equal(smp, mp[order]), seed
    unused = (-50.0, -40.0, 3000.0, 2000.0, 100.0, 100.0, 10.0, 10.0)
    table = [unused, R.cams[2], R.cams[0], R.cams[1]]
    remap = np.array([2, 3, 1], np.int32)[R.frame_cam]
    tmp, tnm, err, _ = sbp_cams(pairs, T, cams=table, frame_cam=dev(remap))
    assert err is None and np.array_equal(tnm, nm) and np.array_equal(tmp, mp)


def test_eight_geometries_in_one_table(gpu_required):
    """every frame its own camera, ORBFE_MULTI_MAX_GROUPS distinct ones: each camera variant moves and widens its frame's
    bounds and changes its intrinsics; each pair equals the single-geometry entry with its Current frame's variant"""
    R = rig()
    limit = fe.ORBFE_MULTI_MAX_GROUPS
    var = []
    for k in range(limit):
        x0, y0, x1, y1, fx, fy, cx, cy = R.cams[min(k // B, len(CAMERAS) - 1)]
        var.append((x0 - 3.25 * k, y0 - 1.5 * k, x1 + 7.5 * k, y1 + 2.25 * k, fx * (1 + 0.002 * k), fy * (1 - 0.001 * k),
                    cx + 0.5 * k, cy - 0.25 * k))
    assert len(set(var)) == limit
    fcam = np.minimum(np.arange(R.F), limit - 1).astype(np.int32)   # frame 8 shares camera 7 with frame 7
    pairs = sbp_pairs()
    T = poses(pairs)
    mp, nm, err, _ = sbp_cams(pairs, T, cams=var, frame_cam=dev(fcam))
    assert err is None
    want_mp, want_nm = sbp_want(pairs, T, cam_of=lambda f: var[fcam[f]])
    assert np.array_equal(nm, want_nm) and np.array_equal(mp, want_mp)


# ---------------------------------------------------------------------------------------------------------------------
# a bad camera index
# ---------------------------------------------------------------------------------------------------------------------
def overflow_store():
    """the rig's store with two more frames: 1000 level-0 keypoints in one grid cell (frame F) and 1000 map points that
    all project into it (frame F + 1), so the pair (F, F + 1) needs 10^6 candidate entries, past its 64 * cap"""
    torch, d = _torch()
    R = rig()
    kps = np.zeros((2, R.cap), fe.KP_DTYPE)
    n = R.cap
    kps["x"], kps["y"] = F32(640.5) + (np.arange(R.cap) % 5).astype(F32) * F32(0.25), F32(360.5)
    kps["size"], kps["angle"], kps["response"] = 31, 10, 1
    desc = np.random.default_rng(3).integers(0, 256, (2, R.cap, 32)).astype(np.uint8)
    _, _, _, _, fx, fy, cx, cy = R.cams[1]
    world = np.zeros((2, R.cap, 3), F32)
    world[1, :, 0] = (F32(640.5) - F32(cx)) / F32(fx) * F32(4)
    world[1, :, 1] = (F32(360.5) - F32(cy)) / F32(fy) * F32(4)
    world[1, :, 2] = 4
    cat = lambda a, b: torch.cat([a, dev(b)]).contiguous()
    return dict(kps=cat(R.kps, kps.view(np.uint8).reshape(2, R.cap, 28)), desc=cat(R.desc, desc),
                cnt=cat(R.cnt, np.array([n, n], np.int32)), world=cat(R.d_world, world),
                flags=cat(R.d_flags, np.ones((2, R.cap), np.uint8)))


@pytest.mark.parametrize("overflow", [False, True], ids=["alone", "beside_overflow"])
@pytest.mark.parametrize("bad", [-1, 3, 1 << 30])
def test_bad_camera_index(gpu_required, bad, overflow):
    """frame 4's camera index is `bad`: the pair that searches it gets nmatches -1 and an untouched row, every other pair
    equals the single-geometry entry, sync reports ORBFE_ERR_ARG; also when another pair of the launch overflows the
    candidate scratch (its nmatches is -1 too)"""
    torch, d = _torch()
    R = rig()
    pairs = sbp_pairs()
    T = poses(pairs)
    fcam = R.frame_cam.copy()
    fcam[4] = bad
    S = overflow_store() if overflow else None
    if overflow:
        pairs = pairs + [(R.F, R.F + 1)]
        T = np.concatenate([T, np.array([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]], F32)])
        fcam = np.concatenate([fcam, [1, 1]]).astype(np.int32)
    P = len(pairs)
    mp0 = np.full((P, R.cap), -1, np.int32)
    mp0[:, 1::4] = 33
    d_mp, d_nm = dev(mp0), torch.full((P,), -9, dtype=torch.int32, device=d)
    src = S or dict(kps=R.kps, desc=R.desc, cnt=R.cnt, world=R.d_world, flags=R.d_flags)
    a = [dev(np.array([c for c, _ in pairs], np.int32)), dev(np.array([l for _, l in pairs], np.int32)), dev(T), dev(fcam)]
    m = fe.ORBmatcher(0.9, True)
    try:
        M.search_by_projection_cams_device(m, P, src["kps"].data_ptr(), src["desc"].data_ptr(), src["cnt"].data_ptr(), R.cap,
                                           a[0].data_ptr(), a[1].data_ptr(), src["world"].data_ptr(), src["flags"].data_ptr(),
                                           a[2].data_ptr(), R.cams, a[3].data_ptr(), 1.2, 8, TH, d_mp.data_ptr(), d_nm.data_ptr())
        err = sync_error(m)
        assert err is not None and err.code == fe.ORBFE_ERR_ARG and "camera index" in str(err), err
        m.sync()   # the flags were cleared
    finally:
        m.close()
    mp, nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
    hit = [j for j, (c, _) in enumerate(pairs) if c == 4]
    assert hit and (nm[hit] == -1).all() and (mp[hit] == mp0[hit]).all()
    if overflow:
        assert nm[-1] == -1
    rest = [j for j in range(len(sbp_pairs())) if j not in hit]
    want_mp, want_nm = sbp_want([pairs[j] for j in rest], T[rest], mp0=mp0[rest])
    assert np.array_equal(nm[rest], want_nm) and np.array_equal(mp[rest], want_mp)


def test_overflow_alone_still_reports_capacity(gpu_required):
    """without a bad camera the overflowing pair of a camera-table launch reports ORBFE_ERR_CAPACITY, as the
    single-geometry entry does"""
    torch, d = _torch()
    R = rig()
    S = overflow_store()
    d_mp, d_nm = dev(np.full((1, R.cap), -1, np.int32)), torch.full((1,), -9, dtype=torch.int32, device=d)
    a = [dev(np.array([R.F], np.int32)), dev(np.array([R.F + 1], np.int32)), dev(np.array([[1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]], F32)),
         dev(np.concatenate([R.frame_cam, [1, 1]]).astype(np.int32))]
    m = fe.ORBmatcher(0.9, True)
    try:
        M.search_by_projection_cams_device(m, 1, S["kps"].data_ptr(), S["desc"].data_ptr(), S["cnt"].data_ptr(), R.cap, a[0].data_ptr(),
                                           a[1].data_ptr(), S["world"].data_ptr(), S["flags"].data_ptr(), a[2].data_ptr(), R.cams,
                                           a[3].data_ptr(), 1.2, 8, TH, d_mp.data_ptr(), d_nm.data_ptr())
        err = sync_error(m)
    finally:
        m.close()
    assert err is not None and err.code == fe.ORBFE_ERR_CAPACITY, err
    assert d_nm.cpu().numpy()[0] == -1


# ---------------------------------------------------------------------------------------------------------------------
# stream order
# ---------------------------------------------------------------------------------------------------------------------
def test_cams_call_on_a_caller_stream_sees_the_previous_call(gpu_required):
    """a single-geometry call on stream A behind a bounded spin writes the 1080p pairs' rows; a camera-table call on
    stream B reads them as occupied slots.  The result equals the two calls run one after the other, and each call adds
    one launch."""
    torch, d = _torch()
    R = rig()
    pairs = sbp_pairs()
    T = poses(pairs)
    first = [0, 1, 2]
    assert all(R.frame_cam[pairs[j][0]] == 0 for j in first)
    # expected: the single-geometry call on the 1080p pairs, then the camera-table call on every pair with those rows
    m1, _ = sbp_single([pairs[j] for j in first], T[first], R.cams[0])
    mp0 = np.full((len(pairs), R.cap), -1, np.int32)
    mp0[first] = m1
    want_mp, want_nm, err, _ = sbp_cams(pairs, T, mp0=mp0)
    assert err is None
    d_mp = dev(np.full((len(pairs), R.cap), -1, np.int32))
    d_nm1 = torch.full((3,), -9, dtype=torch.int32, device=d)
    d_nm = torch.full((len(pairs),), -9, dtype=torch.int32, device=d)
    a, b = torch.cuda.Stream(device=d), torch.cuda.Stream(device=d)
    args = [dev(np.array([c for c, _ in pairs], np.int32)), dev(np.array([l for _, l in pairs], np.int32)), dev(T)]
    torch.cuda.synchronize()
    m = fe.ORBmatcher(0.9, True)
    try:
        x0, y0, x1, y1, fx, fy, cx, cy = R.cams[0]
        with torch.cuda.stream(a):
            torch.cuda._sleep(SPIN)
        n0 = counters(m)
        rc = M._bind().orbfe_search_by_projection_device(m.handle, 3, *R.store(), R.cap, vp(args[0]), vp(args[1]), vp(R.d_world),
                                                         vp(R.d_flags), vp(args[2]), x0, y0, x1, y1, 1.2, 8, fx, fy, cx, cy, TH, 1,
                                                         vp(d_mp), vp(d_nm1), C.c_void_p(a.cuda_stream))
        assert rc == 0 and counters(m) == n0 + 1
        M.search_by_projection_cams_device(m, len(pairs), *[x.value for x in R.store()], R.cap, args[0].data_ptr(), args[1].data_ptr(),
                                           R.d_world.data_ptr(), R.d_flags.data_ptr(), args[2].data_ptr(), R.cams,
                                           R.d_frame_cam.data_ptr(), 1.2, 8, TH, d_mp.data_ptr(), d_nm.data_ptr(), b.cuda_stream)
        assert counters(m) == n0 + 2
        b.synchronize()
        got_mp, got_nm = d_mp.cpu().numpy(), d_nm.cpu().numpy()
        m.sync()
    finally:
        torch.cuda.synchronize()
        m.close()
    assert np.array_equal(got_nm, want_nm) and np.array_equal(got_mp, want_mp)
