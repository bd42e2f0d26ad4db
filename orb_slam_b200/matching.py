"""ctypes views for the array-level matcher entry points (include/orbfe_match.h).

`FrameView` is the slice of ORB_SLAM::Frame (reference include/Frame.h, src/Frame.cc:56-125) that
ORBmatcher reads: undistorted keypoints, descriptors, image bounds, grid cell sizes and per-level scale
factors.  Zero lens distortion is assumed here (mvKeysUn == mvKeys, Frame.cc:291-295), which is what the
synthetic bench uses; the C++ facade passes whatever the real Frame holds.
"""
import ctypes as C

import numpy as np

from . import KP_DTYPE, ORBmatcher, OrbfeError, lib

GRID_COLS, GRID_ROWS = 64, 48  # Frame.h:35-36


class _FrameViewC(C.Structure):
    _fields_ = [("n", C.c_int), ("keys_un", C.c_void_p), ("desc", C.c_void_p),
                ("min_x", C.c_float), ("min_y", C.c_float), ("max_x", C.c_float), ("max_y", C.c_float),
                ("grid_inv_w", C.c_float), ("grid_inv_h", C.c_float),
                ("nlevels", C.c_int), ("scale_factors", C.c_void_p)]


_bound = False


def _bind():
    global _bound
    if _bound:
        return lib()
    L = lib()
    vp = C.c_void_p
    L.orbfe_frame_scale_factors.argtypes = [C.c_float, C.c_int, vp]
    L.orbfe_frame_scale_factors.restype = None
    L.orbfe_search_by_projection_frames.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_float, C.c_float,
                                                    C.c_float, C.c_float, C.c_float, C.c_int, vp, vp]
    L.orbfe_search_by_projection_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp,
                                                    C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                                    C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, vp, vp, vp]
    L.orbfe_guided_search_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int,
                                             C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_int, C.c_int,
                                             vp, vp, vp]
    L.orbfe_search_for_initialization_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, C.c_float, C.c_float, C.c_float,
                                                         C.c_float, C.c_int, C.c_float, C.c_int, vp, vp, vp]
    L.orbfe_undistort_keypoints_device.argtypes = [vp, vp, vp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp]
    L.orbfe_undistort_keypoints.argtypes = [vp, vp, vp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, vp]
    L.orbfe_image_bounds.argtypes = [vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp]
    L.orbfe_search_local_points.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, C.c_float, C.c_float, vp, vp]
    L.orbfe_search_by_projection_kf.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float,
                                                C.c_float, C.c_float, C.c_int, C.c_int, vp, vp]
    L.orbfe_search_by_projection_f1f2.argtypes = [vp, vp, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                                  C.c_float, vp, vp]
    L.orbfe_search_by_bow.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp,
                                      C.c_float, C.c_int, vp, vp]
    L.orbfe_guided_search.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_float, C.c_int, C.c_int, vp, vp]
    L.orbfe_search_for_triangulation.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp,
                                                 vp, vp, C.c_int, vp, vp]
    L.orbfe_guided_best.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int, vp]
    L.orbfe_window_search.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, vp, vp]
    L.orbfe_search_for_initialization.argtypes = [vp, vp, vp, vp, C.c_int, C.c_float, C.c_int, vp, vp]
    L.orbfe_search_by_bow_device.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, C.c_float, C.c_int,
                                             vp, vp, vp]
    L.orbfe_search_for_triangulation_device.argtypes = [vp, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int,
                                                        C.c_int, vp, vp, vp]
    _bound = True
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class FrameView:
    def __init__(self, kps, desc, width, height, scale_factor=1.2, nlevels=8):
        L = _bind()
        self.kps = np.ascontiguousarray(kps, dtype=KP_DTYPE)
        self.desc = np.ascontiguousarray(desc, dtype=np.uint8).reshape(-1, 32)
        self.n = int(self.kps.shape[0])
        self.sf = np.empty(nlevels, np.float32)
        L.orbfe_frame_scale_factors(scale_factor, nlevels, _p(self.sf))
        c = _FrameViewC()
        c.n = self.n
        c.keys_un = self.kps.ctypes.data
        c.desc = self.desc.ctypes.data
        c.min_x, c.min_y, c.max_x, c.max_y = 0.0, 0.0, float(width), float(height)  # Frame.cc:342-348
        c.grid_inv_w = np.float32(GRID_COLS) / np.float32(width)   # Frame.cc:77
        c.grid_inv_h = np.float32(GRID_ROWS) / np.float32(height)  # Frame.cc:78
        c.nlevels = nlevels
        c.scale_factors = self.sf.ctypes.data
        self.c = c


# numpy mirror of OrbfeFrameView (include/orbfe_match.h): lets a whole batch of views be filled with array operations
FRAME_VIEW_DTYPE = np.dtype([("n", "<i4"), ("keys_un", "<u8"), ("desc", "<u8"), ("min_x", "<f4"), ("min_y", "<f4"),
                             ("max_x", "<f4"), ("max_y", "<f4"), ("grid_inv_w", "<f4"), ("grid_inv_h", "<f4"),
                             ("nlevels", "<i4"), ("scale_factors", "<u8")], align=True)
assert FRAME_VIEW_DTYPE.itemsize == C.sizeof(_FrameViewC)
assert all(FRAME_VIEW_DTYPE.fields[f][1] == getattr(_FrameViewC, f).offset for f, _ in _FrameViewC._fields_)


class FrameViewBatch:
    """The views of a batch of frames that live in one (B, cap) keypoint array and one (B, cap, 32) descriptor array --
    the layout orbfe_extract_batch writes.  Same content as B `FrameView`s, built without a Python loop."""

    def __init__(self, kps, desc, counts, width, height, scale_factor=1.2, nlevels=8):
        L = _bind()
        assert kps.dtype == KP_DTYPE and kps.ndim == 2 and kps.strides[1] == KP_DTYPE.itemsize
        assert desc.dtype == np.uint8 and desc.shape[:2] == kps.shape and desc.strides[1] == 32
        self.kps, self.desc = kps, desc
        self.counts = np.ascontiguousarray(counts, np.int32)
        B = kps.shape[0]
        self.sf = np.empty(nlevels, np.float32)
        L.orbfe_frame_scale_factors(scale_factor, nlevels, _p(self.sf))
        v = np.zeros(B, FRAME_VIEW_DTYPE)
        idx = np.arange(B, dtype=np.uint64)
        v["n"] = self.counts
        v["keys_un"] = np.uint64(kps.ctypes.data) + idx * np.uint64(kps.strides[0])
        v["desc"] = np.uint64(desc.ctypes.data) + idx * np.uint64(desc.strides[0])
        v["max_x"], v["max_y"] = float(width), float(height)                        # Frame.cc:342-348
        v["grid_inv_w"] = np.float32(GRID_COLS) / np.float32(width)                 # Frame.cc:77
        v["grid_inv_h"] = np.float32(GRID_ROWS) / np.float32(height)                # Frame.cc:78
        v["nlevels"] = nlevels
        v["scale_factors"] = self.sf.ctypes.data
        self.views = v

    def __len__(self):
        return len(self.views)

    def tail(self):
        """A private copy of the last frame (for the next batch's first pair): (view[1], keep-alive tuple)."""
        i = len(self.views) - 1
        k, d = self.kps[i].copy(), self.desc[i].copy()
        v = self.views[i:i + 1].copy()
        v["keys_un"], v["desc"] = k.ctypes.data, d.ctypes.data
        return v, (k, d, self.sf)


def row_pointers(a):
    """Host addresses of the rows of a 2-D+ array (uint64), for the pointer-array arguments of the batched entry points."""
    return np.uint64(a.ctypes.data) + np.arange(a.shape[0], dtype=np.uint64) * np.uint64(a.strides[0])


def search_by_projection_views(matcher: ORBmatcher, views_cur, views_last, has_ptrs, outlier_ptrs, world_ptrs, Tcws,
                               fx, fy, cx, cy, th, cur_mp):
    """orbfe_search_by_projection_frames on prebuilt argument arrays: `views_*` are FRAME_VIEW_DTYPE arrays, `*_ptrs`
    uint64 arrays of host addresses (one per pair), `Tcws` a contiguous (n, 12) float32 array, `cur_mp` a (n, cap) int32
    array (in: occupied slots >= 0, out: matches).  Returns nmatches[n]."""
    L = _bind()
    n = len(views_cur)
    vc, vl = np.ascontiguousarray(views_cur), np.ascontiguousarray(views_last)
    ptrs = [np.ascontiguousarray(a, np.uint64) for a in (has_ptrs, outlier_ptrs, world_ptrs, row_pointers(Tcws), row_pointers(cur_mp))]
    assert all(len(a) == n for a in ptrs) and len(vl) == n and Tcws.dtype == np.float32 and cur_mp.dtype == np.int32
    nm = np.zeros(n, np.int32)
    _check(L.orbfe_search_by_projection_frames(matcher.handle, n, _p(vc), _p(vl), _p(ptrs[0]), _p(ptrs[1]), _p(ptrs[2]),
                                               _p(ptrs[3]), fx, fy, cx, cy, th, int(matcher.mbCheckOrientation), _p(ptrs[4]), _p(nm)))
    return nm


def _check(rc):
    if rc != 0:
        raise OrbfeError(rc, lib().orbfe_last_error().decode("utf-8", "replace") or "matcher call failed")


def search_by_projection_frames(matcher: ORBmatcher, curs, lasts, last_has_mp, last_outlier, last_world, Tcws,
                                fx, fy, cx, cy, th, cur_mp=None):
    """Batched ORBmatcher::SearchByProjection(CurrentFrame, LastFrame, th) (ORBmatcher.cc:1507-1620).

    curs/lasts: lists of FrameView; last_*: lists of arrays; Tcws: list of 3x4 float arrays.
    Returns (nmatches[npairs], [cur_mp arrays])."""
    L = _bind()
    n = len(curs)
    views_c = (_FrameViewC * n)(*[f.c for f in curs])
    views_l = (_FrameViewC * n)(*[f.c for f in lasts])
    has = [np.ascontiguousarray(a, np.uint8) for a in last_has_mp]
    outl = [np.ascontiguousarray(a, np.uint8) for a in last_outlier]
    world = [np.ascontiguousarray(a, np.float32) for a in last_world]
    T = [np.ascontiguousarray(a, np.float32) for a in Tcws]
    mp = [np.full(f.n, -1, np.int32) if cur_mp is None else np.ascontiguousarray(cur_mp[i], np.int32).copy()
          for i, f in enumerate(curs)]
    arr = lambda xs: (C.c_void_p * n)(*[x.ctypes.data for x in xs])
    nm = np.zeros(n, np.int32)
    _check(L.orbfe_search_by_projection_frames(matcher.handle, n, views_c, views_l, arr(has), arr(outl), arr(world),
                                               arr(T), fx, fy, cx, cy, th, int(matcher.mbCheckOrientation), arr(mp), _p(nm)))
    return nm, mp


def window_search(matcher: ORBmatcher, f1, f2, f1_has_mp, window, min_level=-1, max_level=2 ** 31 - 1):
    L = _bind()
    has = np.ascontiguousarray(f1_has_mp, np.uint8)
    m21 = np.full(max(f2.n, 1), -1, np.int32)
    nm = C.c_int(0)
    _check(L.orbfe_window_search(matcher.handle, C.byref(f1.c), C.byref(f2.c), _p(has), window, min_level, max_level,
                                 float(matcher.mfNNratio), int(matcher.mbCheckOrientation), _p(m21), C.byref(nm)))
    return nm.value, m21[:f2.n]


def search_for_initialization(matcher: ORBmatcher, f1, f2, prev_matched, window):
    L = _bind()
    prev = np.ascontiguousarray(prev_matched, np.float32).copy()
    m12 = np.full(max(f1.n, 1), -1, np.int32)
    nm = C.c_int(0)
    _check(L.orbfe_search_for_initialization(matcher.handle, C.byref(f1.c), C.byref(f2.c), _p(prev), window,
                                             float(matcher.mfNNratio), int(matcher.mbCheckOrientation), _p(m12), C.byref(nm)))
    return nm.value, m12[:f1.n], prev


def search_by_projection_device(matcher: ORBmatcher, npairs, d_kps, d_desc, d_counts, cap, d_cur_idx, d_last_idx, d_world,
                                d_flags, d_Tcw, width, height, scale_factor, nlevels, fx, fy, cx, cy, th, d_cur_mp,
                                d_nmatches, stream=0):
    """Device-pointer form (ints = raw device addresses) of SearchByProjection(Current, Last, th); see
    include/orbfe_match.h.  Zero distortion image bounds (0, 0, width, height) as in Frame.cc:342-348."""
    L = _bind()
    vp = C.c_void_p
    _check(L.orbfe_search_by_projection_device(matcher.handle, npairs, vp(d_kps), vp(d_desc), vp(d_counts), cap,
                                               vp(d_cur_idx), vp(d_last_idx), vp(d_world), vp(d_flags), vp(d_Tcw),
                                               0.0, 0.0, float(width), float(height), scale_factor, nlevels,
                                               fx, fy, cx, cy, th, int(matcher.mbCheckOrientation), vp(d_cur_mp),
                                               vp(d_nmatches), vp(stream)))


def guided_search_device(matcher: ORBmatcher, njobs, d_kps, d_desc, d_counts, cap, d_frame_idx, d_qu, d_qv, d_qr, d_qlo, d_qhi,
                         d_qdesc, d_qangle, d_q_base, d_q_cnt, qcap, width, height, rule, th_dist, d_slot_owner, d_nmatches,
                         stream=0):
    """Device-pointer form of the guided-search skeleton (explicit query windows); see include/orbfe_match.h."""
    L = _bind()
    vp = C.c_void_p
    _check(L.orbfe_guided_search_device(matcher.handle, njobs, vp(d_kps), vp(d_desc), vp(d_counts), cap, vp(d_frame_idx),
                                        vp(d_qu), vp(d_qv), vp(d_qr), vp(d_qlo), vp(d_qhi), vp(d_qdesc), vp(d_qangle),
                                        vp(d_q_base), vp(d_q_cnt), qcap, 0.0, 0.0, float(width), float(height), rule,
                                        float(matcher.mfNNratio), th_dist, int(matcher.mbCheckOrientation), vp(d_slot_owner),
                                        vp(d_nmatches), vp(stream)))


def search_local_points(matcher: ORBmatcher, f, in_view, proj_xy, level, view_cos, desc, th, f_mp=None):
    """ORBmatcher::SearchByProjection(Frame&, const vector<MapPoint*>&, th) on arrays (ORBmatcher.cc:49-125)."""
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    in_view, proj_xy, level, view_cos, desc = a(in_view, np.uint8), a(proj_xy, np.float32), a(level, np.int32), a(view_cos, np.float32), a(desc, np.uint8)
    mp = np.full(max(f.n, 1), -1, np.int32) if f_mp is None else a(f_mp, np.int32).copy()
    nm = C.c_int(0)
    _check(L.orbfe_search_local_points(matcher.handle, C.byref(f.c), len(in_view), _p(in_view), _p(proj_xy), _p(level), _p(view_cos),
                                       _p(desc), th, float(matcher.mfNNratio), _p(mp), C.byref(nm)))
    return nm.value, mp[:f.n]


def search_by_projection_kf(matcher: ORBmatcher, cur, valid, world, min_dist, desc, kf_angle, Tcw, fx, fy, cx, cy, th, orb_dist,
                            cur_mp=None):
    """ORBmatcher::SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) on arrays (ORBmatcher.cc:1622-1746)."""
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    valid, world, min_dist, desc, kf_angle, Tcw = a(valid, np.uint8), a(world, np.float32), a(min_dist, np.float32), a(desc, np.uint8), a(kf_angle, np.float32), a(Tcw, np.float32)
    mp = np.full(max(cur.n, 1), -1, np.int32) if cur_mp is None else a(cur_mp, np.int32).copy()
    nm = C.c_int(0)
    _check(L.orbfe_search_by_projection_kf(matcher.handle, C.byref(cur.c), len(valid), _p(valid), _p(world), _p(min_dist), _p(desc),
                                           _p(kf_angle), _p(Tcw), fx, fy, cx, cy, th, orb_dist, int(matcher.mbCheckOrientation),
                                           _p(mp), C.byref(nm)))
    return nm.value, mp[:cur.n]


def search_by_projection_f1f2(matcher: ORBmatcher, f1, f2, valid1, world1, Tc2w, fx, fy, cx, cy, window, f2_mp=None):
    """ORBmatcher::SearchByProjection(Frame &F1, Frame &F2, windowSize, matches2) on arrays (ORBmatcher.cc:519-594)."""
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    valid1, world1, Tc2w = a(valid1, np.uint8), a(world1, np.float32), a(Tc2w, np.float32)
    mp = np.full(max(f2.n, 1), -1, np.int32) if f2_mp is None else a(f2_mp, np.int32).copy()
    nm = C.c_int(0)
    _check(L.orbfe_search_by_projection_f1f2(matcher.handle, C.byref(f1.c), C.byref(f2.c), _p(valid1), _p(world1), _p(Tc2w), fx, fy,
                                             cx, cy, window, float(matcher.mfNNratio), _p(mp), C.byref(nm)))
    return nm.value, mp[:f2.n]


def feature_vector(node_of_feature):
    """DBoW2::FeatureVector of a frame as (ids, ptr, items): ascending node ids, features in index order inside a node."""
    node_of_feature = np.asarray(node_of_feature)
    order = np.argsort(node_of_feature, kind="stable")
    ids, counts = np.unique(node_of_feature, return_counts=True)
    ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    return ids.astype(np.int32), ptr, order.astype(np.int32)


def search_by_bow(matcher: ORBmatcher, variant, desc1, valid1, angle1, fv1, desc2, valid2, angle2, fv2):
    """ORBmatcher::SearchByBoW on arrays (variant 0: KeyFrame vs Frame, 1: KeyFrame vs KeyFrame)."""
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    desc1, desc2 = a(desc1, np.uint8), a(desc2, np.uint8)
    valid1, valid2 = a(valid1, np.uint8), a(valid2, np.uint8)
    angle1, angle2 = a(angle1, np.float32), a(angle2, np.float32)
    i1, p1, t1 = [a(x, np.int32) for x in fv1]
    i2, p2, t2 = [a(x, np.int32) for x in fv2]
    n1, n2 = desc1.shape[0], desc2.shape[0]
    out = np.full(max(n2 if variant == 0 else n1, 1), -1, np.int32)
    nm = C.c_int(0)
    _check(L.orbfe_search_by_bow(matcher.handle, variant, n1, _p(desc1), _p(valid1), _p(angle1), len(i1), _p(i1), _p(p1), _p(t1),
                                 n2, _p(desc2), _p(valid2), _p(angle2), len(i2), _p(i2), _p(p2), _p(t2),
                                 float(matcher.mfNNratio), int(matcher.mbCheckOrientation), _p(out), C.byref(nm)))
    return nm.value, out[:(n2 if variant == 0 else n1)]


def search_by_bow_device(matcher: ORBmatcher, variant, njobs, d_kps, d_desc, d_counts, cap, d_fv_ids, d_fv_ptr, d_fv_items, d_fv_n,
                         d_valid, d_idx1, d_idx2, d_out, d_nmatches, stream=0):
    """Device-pointer form (ints = raw device addresses) of SearchByBoW for `njobs` (side 1, side 2) frame pairs, with the
    FeatureVectors in the layout of bow.feature_vector_device; see include/orbfe_match.h.  Enqueued, not synchronised."""
    L = _bind()
    vp = C.c_void_p
    _check(L.orbfe_search_by_bow_device(matcher.handle, variant, njobs, vp(d_kps), vp(d_desc), vp(d_counts), cap, vp(d_fv_ids),
                                        vp(d_fv_ptr), vp(d_fv_items), vp(d_fv_n), vp(d_valid), vp(d_idx1), vp(d_idx2),
                                        float(matcher.mfNNratio), int(matcher.mbCheckOrientation), vp(d_out), vp(d_nmatches),
                                        vp(stream)))


def guided_search(matcher: ORBmatcher, f, qu, qv, qr, qlo, qhi, qdesc, qangle, rule, th_dist, hist_mode, slot_owner=None):
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    qu, qv, qr, qlo, qhi, qdesc, qangle = a(qu, np.float32), a(qv, np.float32), a(qr, np.float32), a(qlo, np.int32), a(qhi, np.int32), a(qdesc, np.uint8), a(qangle, np.float32)
    so = np.full(max(f.n, 1), -1, np.int32) if slot_owner is None else a(slot_owner, np.int32).copy()
    nm = C.c_int(0)
    _check(L.orbfe_guided_search(matcher.handle, C.byref(f.c), len(qu), _p(qu), _p(qv), _p(qr), _p(qlo), _p(qhi), _p(qdesc), _p(qangle),
                                 rule, float(matcher.mfNNratio), th_dist, hist_mode, _p(so), C.byref(nm)))
    return nm.value, so[:f.n]


def search_for_triangulation(matcher: ORBmatcher, keys1, desc1, has_mp1, fv1, keys2, desc2, has_mp2, fv2, F12, sigma2):
    """ORBmatcher::SearchForTriangulation on arrays (ORBmatcher.cc:852-1014)."""
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    keys1, keys2 = a(keys1, KP_DTYPE), a(keys2, KP_DTYPE)
    desc1, desc2, has_mp1, has_mp2 = a(desc1, np.uint8), a(desc2, np.uint8), a(has_mp1, np.uint8), a(has_mp2, np.uint8)
    i1, p1, t1 = [a(x, np.int32) for x in fv1]
    i2, p2, t2 = [a(x, np.int32) for x in fv2]
    F12, sigma2 = a(F12, np.float32), a(sigma2, np.float32)
    out = np.full(max(len(keys1), 1), -1, np.int32)
    nm = C.c_int(0)
    _check(L.orbfe_search_for_triangulation(matcher.handle, len(keys1), _p(keys1), _p(desc1), _p(has_mp1), len(i1), _p(i1), _p(p1), _p(t1),
                                            len(keys2), _p(keys2), _p(desc2), _p(has_mp2), len(i2), _p(i2), _p(p2), _p(t2),
                                            _p(F12), _p(sigma2), int(matcher.mbCheckOrientation), _p(out), C.byref(nm)))
    return nm.value, out[:len(keys1)]


def search_for_triangulation_device(matcher: ORBmatcher, njobs, d_kps, d_desc, d_counts, cap, d_fv_ids, d_fv_ptr, d_fv_items, d_fv_n,
                                    d_has_mp, d_idx1, d_idx2, d_F12, sigma2, d_match12, d_nmatches, stream=0):
    """Device-pointer form (ints = raw device addresses) of SearchForTriangulation for `njobs` (pKF1, pKF2) frame pairs, with
    the FeatureVectors in the layout of bow.feature_vector_device, d_F12 = njobs x 9 float32 and `sigma2` the per-level
    KeyFrame::GetSigma2 values on the host; see include/orbfe_match.h.  Enqueued, not synchronised."""
    L = _bind()
    vp = C.c_void_p
    sig = np.ascontiguousarray(sigma2, np.float32)
    _check(L.orbfe_search_for_triangulation_device(matcher.handle, njobs, vp(d_kps), vp(d_desc), vp(d_counts), cap, vp(d_fv_ids),
                                                   vp(d_fv_ptr), vp(d_fv_items), vp(d_fv_n), vp(d_has_mp), vp(d_idx1), vp(d_idx2),
                                                   vp(d_F12), _p(sig), len(sig), int(matcher.mbCheckOrientation), vp(d_match12),
                                                   vp(d_nmatches), vp(stream)))


def guided_best(matcher: ORBmatcher, f, qu, qv, qr, qlo, qhi, qdesc, th_dist):
    L = _bind()
    a = lambda x, t: np.ascontiguousarray(x, t)
    qu, qv, qr, qlo, qhi, qdesc = a(qu, np.float32), a(qv, np.float32), a(qr, np.float32), a(qlo, np.int32), a(qhi, np.int32), a(qdesc, np.uint8)
    out = np.full(max(len(qu), 1), -1, np.int32)
    _check(L.orbfe_guided_best(matcher.handle, C.byref(f.c), len(qu), _p(qu), _p(qv), _p(qr), _p(qlo), _p(qhi), _p(qdesc), th_dist, _p(out)))
    return out[:len(qu)]


def undistort_keypoints(matcher: ORBmatcher, kps, fx, fy, cx, cy, dist):
    """Frame::UndistortKeyPoints (reference src/Frame.cc:289-319) on a keypoint array; dist = (k1, k2, p1, p2[, k3])."""
    L = _bind()
    kps = np.ascontiguousarray(kps, KP_DTYPE)
    d = np.zeros(5, np.float32)
    d[:len(dist)] = dist
    out = np.zeros_like(kps)
    _check(L.orbfe_undistort_keypoints(matcher.handle, _p(kps), _p(out), len(kps), fx, fy, cx, cy, _p(d)))
    return out


def undistort_keypoints_device(matcher: ORBmatcher, d_in, d_out, n, fx, fy, cx, cy, dist, stream=0):
    L = _bind()
    d = np.zeros(5, np.float32)
    d[:len(dist)] = dist
    vp = C.c_void_p
    _check(L.orbfe_undistort_keypoints_device(matcher.handle, vp(d_in), vp(d_out), n, fx, fy, cx, cy, _p(d), vp(stream)))


def image_bounds(matcher: ORBmatcher, cols, rows, fx, fy, cx, cy, dist):
    """Frame::ComputeImageBounds (Frame.cc:321-350): (mnMinX, mnMinY, mnMaxX, mnMaxY)."""
    L = _bind()
    d = np.zeros(5, np.float32)
    d[:len(dist)] = dist
    b = np.zeros(4, np.float32)
    _check(L.orbfe_image_bounds(matcher.handle, cols, rows, fx, fy, cx, cy, _p(d), _p(b)))
    return b


def search_for_initialization_device(matcher: ORBmatcher, npairs, d_kps, d_desc, d_counts, cap, d_f1_idx, d_f2_idx, d_prev_matched,
                                     width, height, window, d_match12, d_nmatches, stream=0):
    """orbfe_search_for_initialization_device on raw device addresses (ints); zero distortion: bounds = [0,W] x [0,H]."""
    L = _bind()
    vp = C.c_void_p
    _check(L.orbfe_search_for_initialization_device(matcher.handle, npairs, vp(d_kps), vp(d_desc), vp(d_counts), cap, vp(d_f1_idx), vp(d_f2_idx),
                                                    vp(d_prev_matched), 0.0, 0.0, float(width), float(height), int(window),
                                                    float(matcher.mfNNratio), int(matcher.mbCheckOrientation), vp(d_match12), vp(d_nmatches),
                                                    vp(stream)))
