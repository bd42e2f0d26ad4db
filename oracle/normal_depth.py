"""MapPoint::UpdateNormalAndDepth (src/MapPoint.cc:273-312) for the tests of orbfe_normal_and_depth(_device) (TEST
INFRASTRUCTURE ONLY).

  normal_depth     the oracle's restatement, oracle/orb_oracle_normal_depth.c, compiled here into
                   oracle/liborb_oracle_normal_depth.so with the flags of oracle/Makefile
  RefMap           the reference's own MapPoint / KeyFrame on a scripted map: oracle/ref_shim/ref_map_point.cc compiled into
                   oracle/_ref/libref_map_point.so, linked against libref_orbslam.so (the reference's sources, unmodified),
                   where the reference sources exist; elsewhere the prebuilt library is used as it is
  shim_scale_add   the shim's `x + y*beta` (the MatExpr of `normal + normali/cv::norm(normali)`), from the same library"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborb_oracle_normal_depth.so")
_SRC = os.path.join(_HERE, "orb_oracle_normal_depth.c")
_REF_SO = os.path.join(R._DIR, "libref_map_point.so")
_REF_SRC = os.path.join(_HERE, "ref_shim", "ref_map_point.cc")
_lib = None
_ref_lib = None


def build(force=False):
    """Compile the oracle library, and the reference driver where the reference sources exist (after `make ref`)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                               "-std=gnu11", "-shared", _SRC, "-o", _SO, "-lm"])
    root = R.REFERENCE_ROOT
    if os.path.isdir(os.path.join(root, "src")):
        base = R.build()
        if force or not os.path.exists(_REF_SO) or os.path.getmtime(_REF_SO) < max(os.path.getmtime(_REF_SRC), os.path.getmtime(base)):
            subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC",
                                   "-w", "-shared", "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"),
                                   "-I" + root, _REF_SRC, "-o", _REF_SO, "-L" + R._DIR, "-lref_orbslam", "-Wl,-rpath,$ORIGIN",
                                   "-lpthread"])
    return _SO


def ref_available():
    return os.path.exists(_REF_SO) and R.available()


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, i = C.c_void_p, C.c_int
        L.orb_oracle_normal_depth.argtypes = [i, vp, vp, vp, vp, vp, C.c_float, i, vp, vp, vp, vp]
        L.orb_oracle_normal_depth.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def normal_depth(world, ref_centers, ref_octave, group_ptr, obs_centers, scale_factor, scale_factors, normal=None, min_dist=None,
                 max_dist=None):
    """The oracle on host arrays in the layout of orbfe_normal_and_depth: returns (normal [n,3], min_dist [n], max_dist [n])
    float32; rows of empty groups are those passed in (zeros when not given)."""
    gp = np.ascontiguousarray(group_ptr, np.int32)
    n = len(gp) - 1
    f3 = lambda x: np.ascontiguousarray(x, np.float32).reshape(-1, 3)
    w, rc = f3(world), f3(ref_centers)
    oc = f3(obs_centers) if np.asarray(obs_centers).size else np.zeros((1, 3), np.float32)
    oct_ = np.ascontiguousarray(ref_octave, np.int32)
    sf = np.ascontiguousarray(scale_factors, np.float32)
    on = np.zeros((max(n, 1), 3), np.float32) if normal is None else np.array(f3(normal), copy=True)
    omin = np.zeros(max(n, 1), np.float32) if min_dist is None else np.array(min_dist, np.float32, copy=True)
    omax = np.zeros(max(n, 1), np.float32) if max_dist is None else np.array(max_dist, np.float32, copy=True)
    lib().orb_oracle_normal_depth(n, _p(w), _p(rc), _p(oct_), _p(gp), _p(oc), float(np.float32(scale_factor)), len(sf), _p(sf), _p(on),
                                  _p(omin), _p(omax))
    return on[:n], omin[:n], omax[:n]


def _ref():
    global _ref_lib
    if _ref_lib is None:
        if not os.path.exists(_REF_SO):
            build()
        L = C.CDLL(_REF_SO, mode=os.RTLD_NOW | os.RTLD_LOCAL)
        vp, i = C.c_void_p, C.c_int
        L.ref_nd_create.restype = vp
        L.ref_nd_free.argtypes = [vp]
        L.ref_nd_add_keyframe.argtypes = [vp, vp, vp, i, C.c_float, i, i]
        L.ref_nd_keyframe.argtypes = [vp, i, vp, vp, vp]
        L.ref_nd_add_point.argtypes = [vp, vp, i]
        L.ref_nd_add_observation.argtypes = [vp, i, i, i]
        L.ref_nd_set_point_bad.argtypes = [vp, i]
        L.ref_nd_set_world_pos.argtypes = [vp, i, vp]
        L.ref_nd_update.argtypes = [vp, i]
        L.ref_nd_get.argtypes = [vp, i, vp, vp, vp]
        L.ref_nd_observations.argtypes = [vp, i, vp, vp, i]
        L.ref_shim_scale_add.argtypes = [vp, vp, C.c_double, i, vp]
        L.ref_shim_scale_add.restype = None
        _ref_lib = L
    return _ref_lib


def shim_scale_add(x, y, beta):
    """The shim's `x + y*beta` on float32 columns."""
    x, y = np.ascontiguousarray(x, np.float32).ravel(), np.ascontiguousarray(y, np.float32).ravel()
    out = np.zeros(len(x), np.float32)
    _ref().ref_shim_scale_add(_p(x), _p(y), float(beta), len(x), _p(out))
    return out


class RefMap:
    """A scripted map of the reference's own KeyFrames and MapPoints (ids = creation order)."""

    def __init__(self):
        self.L = _ref()
        self.h = self.L.ref_nd_create()

    def add_keyframe(self, Tcw34, octaves, scale_factor, nlevels, bad=False):
        T = np.ascontiguousarray(Tcw34, np.float32).reshape(3, 4)
        o = np.ascontiguousarray(octaves, np.int32)
        return self.L.ref_nd_add_keyframe(self.h, _p(T), _p(o) if len(o) else None, len(o), float(np.float32(scale_factor)), int(nlevels),
                                          int(bool(bad)))

    def keyframe(self, kf, nlevels):
        """(GetCameraCenter() [3], GetScaleFactor(), [GetScaleFactor(l) for l < nlevels]) as float32."""
        c, s, t = np.zeros(3, np.float32), np.zeros(1, np.float32), np.zeros(max(nlevels, 1), np.float32)
        self.L.ref_nd_keyframe(self.h, kf, _p(c), _p(s), _p(t))
        return c, s[0], t[:nlevels]

    def add_point(self, pos, ref_kf):
        p = np.ascontiguousarray(pos, np.float32)
        return self.L.ref_nd_add_point(self.h, _p(p), ref_kf)

    def add_observation(self, mp, kf, idx):
        self.L.ref_nd_add_observation(self.h, mp, kf, idx)

    def set_point_bad(self, mp):
        self.L.ref_nd_set_point_bad(self.h, mp)

    def set_world_pos(self, mp, pos):
        p = np.ascontiguousarray(pos, np.float32)
        self.L.ref_nd_set_world_pos(self.h, mp, _p(p))

    def update(self, mp):
        """UpdateNormalAndDepth, then (GetNormal() [3], GetMinDistanceInvariance(), GetMaxDistanceInvariance())."""
        self.L.ref_nd_update(self.h, mp)
        return self.get(mp)

    def get(self, mp):
        n, a, b = np.zeros(3, np.float32), np.zeros(1, np.float32), np.zeros(1, np.float32)
        self.L.ref_nd_get(self.h, mp, _p(n), _p(a), _p(b))
        return n, a[0], b[0]

    def observations(self, mp, cap=1 << 16):
        k, i = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        n = self.L.ref_nd_observations(self.h, mp, _p(k), _p(i), cap)
        return list(zip(k[:n].tolist(), i[:n].tolist()))

    def close(self):
        if self.h:
            self.L.ref_nd_free(self.h)
            self.h = None
