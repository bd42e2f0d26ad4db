"""ctypes binding of the CPU ORACLE (oracle/liborb_oracle.so).  TEST INFRASTRUCTURE ONLY.

Importable from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
The product package (orb_slam_b200) must never import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import _cdll

MAX_LEVELS = 32
EDGE = 16
TIES_CANONICAL, TIES_NTH_ELEMENT = 0, 1
TRIG_RN, TRIG_LIBMF = 0, 1
GRID_COLS, GRID_ROWS = 64, 48

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])
assert KP_DTYPE.itemsize == 28


class Params(C.Structure):
    _fields_ = [("nfeatures", C.c_int), ("nlevels", C.c_int), ("score_type", C.c_int), ("fast_th", C.c_int),
                ("scale_factor", C.c_double),
                ("scale", C.c_float * MAX_LEVELS), ("inv_scale", C.c_float * MAX_LEVELS),
                ("quota", C.c_int * MAX_LEVELS), ("umax", C.c_int * 16),
                ("ties_mode", C.c_int), ("trig_mode", C.c_int)]


class CellGrid(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("cols", "rows", "cell_w", "cell_h", "n_cells", "nf_cell", "Wd", "Hd")]


class Dump(C.Structure):
    _fields_ = [("nlevels", C.c_int), ("w", C.c_int * MAX_LEVELS), ("h", C.c_int * MAX_LEVELS),
                ("stride", C.c_size_t * MAX_LEVELS),
                ("level", C.POINTER(C.c_uint8) * MAX_LEVELS), ("blurred", C.POINTER(C.c_uint8) * MAX_LEVELS),
                ("n_level_kp", C.c_int * MAX_LEVELS), ("n_ties_at_cut", C.c_long), ("n_fallback_cells", C.c_long)]


class Frame(C.Structure):
    _fields_ = [("n", C.c_int), ("keys_un", C.c_void_p), ("desc", C.c_void_p),
                ("min_x", C.c_float), ("min_y", C.c_float), ("max_x", C.c_float), ("max_y", C.c_float),
                ("grid_inv_w", C.c_float), ("grid_inv_h", C.c_float),
                ("nlevels", C.c_int), ("scale_factors", C.c_void_p),
                ("cell_start", C.c_int * (GRID_COLS * GRID_ROWS + 1)), ("cell_items", C.c_void_p)]


def build():
    """Bring oracle/liborb_oracle.so up to date with oracle/Makefile (gcc/g++). Building the checker is not using it."""
    subprocess.check_call(["make", "-C", _cdll.HERE, "-s"])
    return os.path.join(_cdll.HERE, "liborb_oracle.so")


def _signatures():
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    P, PI, FR = C.POINTER(Params), C.POINTER(C.c_int), C.POINTER(Frame)
    return {
        "orb_oracle_params_init": (i, [P, i, f, i, i, i]),
        "orb_oracle_level_size": (i, [P, i, i, i, PI, PI]),
        "orb_oracle_cell_grid": (i, [P, i, i, i, i, i, C.POINTER(CellGrid)]),
        "orb_oracle_resize_linear_u8": (None, [vp, i, i, sz, vp, i, i, sz]),
        "orb_oracle_reflect101_frame": (None, [vp, i, i, sz, i]),
        "orb_oracle_fast_m": (i, [vp, sz]),
        "orb_oracle_fast_detect": (i, [vp, i, i, sz, i, vp, vp, vp, i]),
        "orb_oracle_blur7_u8": (None, [vp, i, i, sz, vp, sz]),
        "orb_oracle_fast_atan2": (f, [f, f]),
        "orb_oracle_ic_angle": (f, [vp, sz, vp]),
        "orb_oracle_ic_moments": (None, [vp, sz, vp, PI, PI]),
        "orb_oracle_brief": (None, [vp, sz, f, i, vp]),
        "orb_oracle_extract": (i, [P, vp, i, i, sz, vp, vp, i, PI, C.POINTER(Dump)]),
        "orb_oracle_dump_free": (None, [C.POINTER(Dump)]),
        "orb_oracle_hamming": (i, [vp, vp]),
        "orb_oracle_frame_grid": (None, [FR]),
        "orb_oracle_features_in_area": (i, [FR, f, f, f, i, i, vp, i]),
        "orb_oracle_frame_scale_factors": (None, [f, i, vp]),
        "orb_oracle_three_maxima": (None, [vp, i, PI, PI, PI]),
        "orb_oracle_search_by_projection_ff": (i, [FR, FR, vp, vp, vp, vp, f, f, f, f, f, i, vp]),
        "orb_oracle_window_search": (i, [FR, FR, vp, i, i, i, f, i, vp]),
        "orb_oracle_search_for_initialization": (i, [FR, FR, vp, i, f, i, vp]),
        "orb_oracle_search_local_points": (i, [FR, i, vp, vp, vp, vp, vp, f, f, vp]),
        "orb_oracle_search_by_projection_kf": (i, [FR, i, vp, vp, vp, vp, vp, vp, f, f, f, f, f, i, i, vp]),
        "orb_oracle_search_by_projection_f1f2": (i, [FR, FR, vp, vp, vp, f, f, f, f, i, f, vp]),
        "orb_oracle_guided_search": (i, [FR, i, vp, vp, vp, vp, vp, vp, vp, i, f, i, i, vp]),
        "orb_oracle_search_for_triangulation": (i, [i, vp, vp, vp, i, vp, vp, vp, i, vp, vp, vp, i, vp, vp, vp, vp, vp, i, vp]),
        "orb_oracle_guided_best": (None, [FR, i, vp, vp, vp, vp, vp, vp, i, vp]),
        "orb_oracle_search_by_bow": (i, [i, i, vp, vp, vp, i, vp, vp, vp, i, vp, vp, vp, i, vp, vp, vp, f, i, vp]),
        "orb_oracle_knn2": (None, [vp, i, vp, C.c_long, vp, vp, vp]),
    }


_p = _cdll.p
lib = _cdll.loader("liborb_oracle.so", _signatures())


def make_params(nfeatures=1000, scale_factor=1.2, nlevels=8, score_type=1, fast_th=20,
                ties_mode=TIES_CANONICAL, trig_mode=TRIG_RN):
    p = Params()
    rc = lib().orb_oracle_params_init(C.byref(p), nfeatures, scale_factor, nlevels, score_type, fast_th)
    if rc:
        raise ValueError("orb_oracle_params_init failed: %d" % rc)
    p.ties_mode, p.trig_mode = ties_mode, trig_mode
    return p


def level_size(p, level, W, H):
    w, h = C.c_int(), C.c_int()
    lib().orb_oracle_level_size(C.byref(p), level, W, H, C.byref(w), C.byref(h))
    return w.value, h.value


def cell_grid(p, level, W0, H0, w, h):
    g = CellGrid()
    rc = lib().orb_oracle_cell_grid(C.byref(p), level, W0, H0, w, h, C.byref(g))
    return rc, g


def resize_linear(src, dw, dh):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    dst = np.empty((dh, dw), np.uint8)
    lib().orb_oracle_resize_linear_u8(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dw, dh, dst.strides[0])
    return dst


def reflect101_pad(img, b=EDGE):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape
    buf = np.zeros((h + 2 * b, w + 2 * b), np.uint8)
    buf[b:b + h, b:b + w] = img
    lib().orb_oracle_reflect101_frame(_p(buf), w, h, buf.strides[0], b)
    return buf


def fast_m_map(img):
    """m value of every pixel with a full ring (3-px margin); zero elsewhere. Slow: small images only."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape
    out = np.zeros((h, w), np.int32)
    L = lib()
    base = img.ctypes.data
    for y in range(3, h - 3):
        for x in range(3, w - 3):
            out[y, x] = L.orb_oracle_fast_m(C.c_void_p(base + y * img.strides[0] + x), img.strides[0])
    return out


def fast_detect(img, th):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape
    cap = max(16, (w * h) // 4 + 16)
    xs, ys, sc = (np.empty(cap, np.int32) for _ in range(3))
    n = lib().orb_oracle_fast_detect(_p(img), w, h, img.strides[0], th, _p(xs), _p(ys), _p(sc), cap)
    assert n <= cap
    return xs[:n].copy(), ys[:n].copy(), sc[:n].copy()


def blur7(img):
    """GaussianBlur 7x7 sigma 2 with BORDER_REFLECT_101 (integer 2.4 engine) of a whole image."""
    buf = reflect101_pad(img, 3)
    h, w = img.shape
    dst = np.empty((h, w), np.uint8)
    lib().orb_oracle_blur7_u8(C.c_void_p(buf.ctypes.data + 3 * buf.strides[0] + 3), w, h, buf.strides[0], _p(dst), dst.strides[0])
    return dst


def fast_atan2(y, x):
    return lib().orb_oracle_fast_atan2(float(y), float(x))


UMAX = np.array([15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3], np.int32)


def ic_angle(padded, stride_elems_unused, x, y, pad=EDGE):
    """padded: reflect-101 padded level (pad px); (x, y) in interior coordinates."""
    return lib().orb_oracle_ic_angle(C.c_void_p(padded.ctypes.data + (y + pad) * padded.strides[0] + (x + pad)),
                                     padded.strides[0], _p(UMAX))


def ic_moments(padded, x, y, pad=EDGE):
    m01, m10 = C.c_int(), C.c_int()
    lib().orb_oracle_ic_moments(C.c_void_p(padded.ctypes.data + (y + pad) * padded.strides[0] + (x + pad)),
                                padded.strides[0], _p(UMAX), C.byref(m01), C.byref(m10))
    return m01.value, m10.value


def brief(padded, x, y, angle_deg, trig_mode=TRIG_RN, pad=EDGE):
    d = np.empty(32, np.uint8)
    lib().orb_oracle_brief(C.c_void_p(padded.ctypes.data + (y + pad) * padded.strides[0] + (x + pad)),
                           padded.strides[0], float(angle_deg), trig_mode, _p(d))
    return d


def extract(p, img, cap=None, want_dump=False):
    """ORBextractor::operator(): returns (rc, keypoints[KP_DTYPE], descriptors[N,32], dump or None).

    dump = dict(levels=[unblurred interior arrays], blurred=[...], n_level_kp=[...], ties=int, fallback=int)
    """
    img = np.ascontiguousarray(img, dtype=np.uint8)
    H, W = img.shape
    cap = cap or max(p.nfeatures, 1)
    kps = np.zeros(cap, KP_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    n = C.c_int(0)
    d = Dump() if want_dump else None
    rc = lib().orb_oracle_extract(C.byref(p), _p(img), W, H, img.strides[0], _p(kps), _p(desc), cap, C.byref(n),
                                  C.byref(d) if want_dump else None)
    out = None
    if want_dump and rc in (0, -3):
        out = {"levels": [], "blurred": [], "n_level_kp": [], "ties": d.n_ties_at_cut, "fallback": d.n_fallback_cells}
        for l in range(d.nlevels):
            w, h, s = d.w[l], d.h[l], d.stride[l]
            for key, ptr in (("levels", d.level[l]), ("blurred", d.blurred[l])):
                full = np.ctypeslib.as_array(ptr, shape=(h + 2 * EDGE, s)).copy()
                out[key].append(full[:, :w + 2 * EDGE])
            out["n_level_kp"].append(d.n_level_kp[l])
    if want_dump:
        lib().orb_oracle_dump_free(C.byref(d))
    m = min(n.value, cap)
    return rc, kps[:m].copy(), desc[:m].copy(), out


def hamming(a, b):
    a = np.ascontiguousarray(a, np.uint8)
    b = np.ascontiguousarray(b, np.uint8)
    return lib().orb_oracle_hamming(_p(a), _p(b))


def knn2(q, db):
    q = np.ascontiguousarray(q, np.uint8)
    db = np.ascontiguousarray(db, np.uint8)
    nq, ndb = q.shape[0], db.shape[0]
    bd, bi, sd = (np.empty(nq, np.int32) for _ in range(3))
    lib().orb_oracle_knn2(_p(q), nq, _p(db), ndb, _p(bd), _p(bi), _p(sd))
    return bd, bi, sd


class OracleFrame:
    """The slice of ORB_SLAM::Frame the matchers read (Frame.cc:56-125), zero distortion."""

    def __init__(self, kps, desc, width, height, scale_factor=1.2, nlevels=8):
        self.kps = np.ascontiguousarray(kps, dtype=KP_DTYPE)
        self.desc = np.ascontiguousarray(desc, dtype=np.uint8)
        self.n = int(self.kps.shape[0])
        self.sf = np.empty(nlevels, np.float32)
        lib().orb_oracle_frame_scale_factors(scale_factor, nlevels, _p(self.sf))
        self.items = np.zeros(max(self.n, 1), np.int32)
        f = Frame()
        f.n = self.n
        f.keys_un = self.kps.ctypes.data
        f.desc = self.desc.ctypes.data
        f.min_x, f.min_y, f.max_x, f.max_y = 0.0, 0.0, float(width), float(height)  # Frame.cc:342-348
        f.grid_inv_w = np.float32(GRID_COLS) / np.float32(width)   # Frame.cc:77
        f.grid_inv_h = np.float32(GRID_ROWS) / np.float32(height)  # Frame.cc:78
        f.nlevels = nlevels
        f.scale_factors = self.sf.ctypes.data
        f.cell_items = self.items.ctypes.data
        self.c = f
        lib().orb_oracle_frame_grid(C.byref(f))

    def features_in_area(self, x, y, r, min_level, max_level):
        out = np.empty(max(self.n, 1), np.int32)
        n = lib().orb_oracle_features_in_area(C.byref(self.c), x, y, r, min_level, max_level, _p(out), self.n)
        return out[:n].copy()


def search_by_projection_ff(cur, last, last_has_mp, last_outlier, last_world, Tcw, fx, fy, cx, cy, th,
                            check_orientation=True, cur_mp=None):
    cur_mp = np.full(cur.n, -1, np.int32) if cur_mp is None else np.ascontiguousarray(cur_mp, np.int32).copy()
    has = np.ascontiguousarray(last_has_mp, np.uint8)
    outl = np.ascontiguousarray(last_outlier, np.uint8)
    world = np.ascontiguousarray(last_world, np.float32)
    T = np.ascontiguousarray(Tcw, np.float32)
    n = lib().orb_oracle_search_by_projection_ff(C.byref(cur.c), C.byref(last.c), _p(has), _p(outl), _p(world), _p(T),
                                                 fx, fy, cx, cy, th, int(check_orientation), _p(cur_mp))
    return n, cur_mp


def window_search(f1, f2, f1_has_mp, window, min_level=-1, max_level=2 ** 31 - 1, nnratio=0.6, check_orientation=True):
    has = np.ascontiguousarray(f1_has_mp, np.uint8)
    m21 = np.empty(max(f2.n, 1), np.int32)
    n = lib().orb_oracle_window_search(C.byref(f1.c), C.byref(f2.c), _p(has), window, min_level, max_level, nnratio,
                                       int(check_orientation), _p(m21))
    return n, m21[:f2.n]


def search_for_initialization(f1, f2, prev_matched, window, nnratio=0.9, check_orientation=True):
    prev = np.ascontiguousarray(prev_matched, np.float32).copy()
    m12 = np.empty(max(f1.n, 1), np.int32)
    n = lib().orb_oracle_search_for_initialization(C.byref(f1.c), C.byref(f2.c), _p(prev), window, nnratio,
                                                   int(check_orientation), _p(m12))
    return n, m12[:f1.n], prev


def _a(x, t):
    return np.ascontiguousarray(x, t)


def search_local_points(f, in_view, proj_xy, level, view_cos, desc, th, nnratio=0.8, f_mp=None):
    mp = np.full(max(f.n, 1), -1, np.int32) if f_mp is None else _a(f_mp, np.int32).copy()
    iv, pj, lv, vc, ds = _a(in_view, np.uint8), _a(proj_xy, np.float32), _a(level, np.int32), _a(view_cos, np.float32), _a(desc, np.uint8)
    n = lib().orb_oracle_search_local_points(C.byref(f.c), len(iv), _p(iv), _p(pj), _p(lv), _p(vc), _p(ds), th, nnratio, _p(mp))
    return n, mp[:f.n]


def search_by_projection_kf(cur, valid, world, min_dist, desc, kf_angle, Tcw, fx, fy, cx, cy, th, orb_dist, check_orientation=True,
                            cur_mp=None):
    mp = np.full(max(cur.n, 1), -1, np.int32) if cur_mp is None else _a(cur_mp, np.int32).copy()
    v, w, md, ds, ka, T = _a(valid, np.uint8), _a(world, np.float32), _a(min_dist, np.float32), _a(desc, np.uint8), _a(kf_angle, np.float32), _a(Tcw, np.float32)
    n = lib().orb_oracle_search_by_projection_kf(C.byref(cur.c), len(v), _p(v), _p(w), _p(md), _p(ds), _p(ka), _p(T), fx, fy, cx, cy,
                                                 th, orb_dist, int(check_orientation), _p(mp))
    return n, mp[:cur.n]


def search_by_projection_f1f2(f1, f2, valid1, world1, Tc2w, fx, fy, cx, cy, window, nnratio=0.9, f2_mp=None):
    mp = np.full(max(f2.n, 1), -1, np.int32) if f2_mp is None else _a(f2_mp, np.int32).copy()
    v, w, T = _a(valid1, np.uint8), _a(world1, np.float32), _a(Tc2w, np.float32)
    n = lib().orb_oracle_search_by_projection_f1f2(C.byref(f1.c), C.byref(f2.c), _p(v), _p(w), _p(T), fx, fy, cx, cy, window, nnratio, _p(mp))
    return n, mp[:f2.n]


def search_by_bow(variant, desc1, valid1, angle1, fv1, desc2, valid2, angle2, fv2, nnratio=0.75, check_orientation=True):
    desc1, desc2 = _a(desc1, np.uint8), _a(desc2, np.uint8)
    valid1, valid2, angle1, angle2 = _a(valid1, np.uint8), _a(valid2, np.uint8), _a(angle1, np.float32), _a(angle2, np.float32)
    i1, p1, t1 = [_a(x, np.int32) for x in fv1]
    i2, p2, t2 = [_a(x, np.int32) for x in fv2]
    n1, n2 = desc1.shape[0], desc2.shape[0]
    out = np.full(max(n2 if variant == 0 else n1, 1), -1, np.int32)
    n = lib().orb_oracle_search_by_bow(variant, n1, _p(desc1), _p(valid1), _p(angle1), len(i1), _p(i1), _p(p1), _p(t1),
                                       n2, _p(desc2), _p(valid2), _p(angle2), len(i2), _p(i2), _p(p2), _p(t2),
                                       nnratio, int(check_orientation), _p(out))
    return n, out[:(n2 if variant == 0 else n1)]


def guided_search(f, qu, qv, qr, qlo, qhi, qdesc, qangle, rule, nnratio, th_dist, hist_mode, slot_owner=None):
    qu, qv, qr, qlo, qhi, qdesc, qangle = _a(qu, np.float32), _a(qv, np.float32), _a(qr, np.float32), _a(qlo, np.int32), _a(qhi, np.int32), _a(qdesc, np.uint8), _a(qangle, np.float32)
    so = np.full(max(f.n, 1), -1, np.int32) if slot_owner is None else _a(slot_owner, np.int32).copy()
    n = lib().orb_oracle_guided_search(C.byref(f.c), len(qu), _p(qu), _p(qv), _p(qr), _p(qlo), _p(qhi), _p(qdesc), _p(qangle), rule,
                                       nnratio, th_dist, hist_mode, _p(so))
    return n, so[:f.n]


def search_for_triangulation(keys1, desc1, has_mp1, fv1, keys2, desc2, has_mp2, fv2, F12, sigma2, check_orientation=True):
    keys1, keys2 = _a(keys1, KP_DTYPE), _a(keys2, KP_DTYPE)
    desc1, desc2, has_mp1, has_mp2 = _a(desc1, np.uint8), _a(desc2, np.uint8), _a(has_mp1, np.uint8), _a(has_mp2, np.uint8)
    i1, p1, t1 = [_a(x, np.int32) for x in fv1]
    i2, p2, t2 = [_a(x, np.int32) for x in fv2]
    F12, sigma2 = _a(F12, np.float32), _a(sigma2, np.float32)
    out = np.full(max(len(keys1), 1), -1, np.int32)
    n = lib().orb_oracle_search_for_triangulation(len(keys1), _p(keys1), _p(desc1), _p(has_mp1), len(i1), _p(i1), _p(p1), _p(t1),
                                                  len(keys2), _p(keys2), _p(desc2), _p(has_mp2), len(i2), _p(i2), _p(p2), _p(t2),
                                                  _p(F12), _p(sigma2), int(check_orientation), _p(out))
    return n, out[:len(keys1)]


def guided_best(f, qu, qv, qr, qlo, qhi, qdesc, th_dist):
    qu, qv, qr, qlo, qhi, qdesc = _a(qu, np.float32), _a(qv, np.float32), _a(qr, np.float32), _a(qlo, np.int32), _a(qhi, np.int32), _a(qdesc, np.uint8)
    out = np.full(max(len(qu), 1), -1, np.int32)
    lib().orb_oracle_guided_best(C.byref(f.c), len(qu), _p(qu), _p(qv), _p(qr), _p(qlo), _p(qhi), _p(qdesc), th_dist, _p(out))
    return out[:len(qu)]


# ---- SURVEY section 8(f) rows N2 / N4 (orb_oracle_bow.c) ----
def bow_descend(voc, desc, levelsup=4):
    """voc: dict(node_desc, child_ptr, children, word_id, weight, L).  Returns (leaf, node) per descriptor."""
    desc = _a(desc, np.uint8)
    n = len(desc)
    leaf, node = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
    f = lib().orb_oracle_bow_descend
    f.restype = None
    f(_p(voc["node_desc"]), _p(voc["child_ptr"]), _p(voc["children"]), C.c_int(voc["L"]), _p(desc), C.c_int(n), C.c_int(levelsup),
      _p(leaf), _p(node))
    return leaf[:n], node[:n]


def bow_transform(voc, desc, levelsup=4, weighting=0, norm=1):
    desc = _a(desc, np.uint8)
    n = len(desc)
    cap = max(n, 1)
    bow_ids, bow_vals = np.zeros(cap, np.int32), np.zeros(cap, np.float64)
    fv_ids, fv_ptr, fv_feats = np.zeros(cap, np.int32), np.zeros(cap + 1, np.int32), np.zeros(cap, np.int32)
    nw, nn = C.c_int(0), C.c_int(0)
    f = lib().orb_oracle_bow_transform
    f.restype = None
    f(_p(voc["node_desc"]), _p(voc["child_ptr"]), _p(voc["children"]), _p(voc["word_id"]), _p(voc["weight"]), C.c_int(voc["L"]),
      C.c_int(weighting), C.c_int(norm), _p(desc), C.c_int(n), C.c_int(levelsup), C.byref(nw), _p(bow_ids), _p(bow_vals),
      C.byref(nn), _p(fv_ids), _p(fv_ptr), _p(fv_feats))
    return (bow_ids[:nw.value], bow_vals[:nw.value]), (fv_ids[:nn.value], fv_ptr[:nn.value + 1], fv_feats[:fv_ptr[nn.value]])


def distinctive_descriptors(desc, group_ptr):
    desc, group_ptr = _a(desc, np.uint8), _a(group_ptr, np.int32)
    ng = len(group_ptr) - 1
    best = np.zeros(max(ng, 1), np.int32)
    f = lib().orb_oracle_distinctive
    f.restype = None
    f(_p(desc), _p(group_ptr), C.c_int(ng), _p(best))
    return best[:ng]


def bow_db_detect(mode, q_ids, q_vals, kf_ptr, db_ids, db_vals, connected, covis_ptr, covis, min_score):
    q_ids, q_vals, kf_ptr = _a(q_ids, np.int32), _a(q_vals, np.float64), _a(kf_ptr, np.int32)
    db_ids, db_vals, covis_ptr, covis = _a(db_ids, np.int32), _a(db_vals, np.float64), _a(covis_ptr, np.int32), _a(covis, np.int32)
    connected = _a(connected, np.uint8)
    nkf = len(kf_ptr) - 1
    cand, common, score = np.zeros(max(nkf, 1), np.int32), np.zeros(max(nkf, 1), np.int32), np.zeros(max(nkf, 1), np.float32)
    f = lib().orb_oracle_bow_db_detect
    f.restype = C.c_int
    n = f(C.c_int(mode), C.c_int(len(q_ids)), _p(q_ids), _p(q_vals), C.c_int(nkf), _p(kf_ptr), _p(db_ids), _p(db_vals), _p(connected),
          _p(covis_ptr), _p(covis), C.c_float(min_score), _p(cand), _p(common), _p(score))
    return cand[:n], common[:nkf], score[:nkf]


# ---- Frame::UndistortKeyPoints / ComputeImageBounds (src/Frame.cc:289-350) ----
def undistort_points(pts, fx, fy, cx, cy, dist):
    pts, dist = _a(pts, np.float32).reshape(-1, 2), _a(dist, np.float32)
    out = np.zeros_like(pts)
    f = lib().orb_oracle_undistort_points
    f.restype = None
    f(_p(pts), C.c_int(len(pts)), C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy), _p(dist), _p(out))
    return out


def undistort_keypoints(kps, fx, fy, cx, cy, dist):
    kps, dist = _a(kps, KP_DTYPE), _a(dist, np.float32)
    out = np.zeros_like(kps)
    f = lib().orb_oracle_undistort_keypoints
    f.restype = None
    f(_p(kps), C.c_int(len(kps)), C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy), _p(dist), _p(out))
    return out


def image_bounds(cols, rows, fx, fy, cx, cy, dist):
    dist = _a(dist, np.float32)
    b = np.zeros(4, np.float32)
    f = lib().orb_oracle_image_bounds
    f.restype = None
    f(C.c_int(cols), C.c_int(rows), C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy), _p(dist), _p(b))
    return b
