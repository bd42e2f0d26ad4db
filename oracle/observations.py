"""MapPoint::GetObservations() of named points as the inverse of the live keyframes' rows, for the tests of
orbfe_covis_observations_device (TEST INFRASTRUCTURE ONLY).

  observations()  the oracle's restatement, oracle/orb_oracle_observations.c, compiled here into
                  oracle/liborb_oracle_observations.so with the flags of oracle/Makefile
  RefObservations the reference's own KeyFrame / MapPoint on a scripted map (oracle.covis.RefCovis) plus MapPoint::Replace,
                  the local-BA outlier erase, the halves of an observation and GetReferenceKeyFrame():
                  oracle/ref_shim/ref_observations.cc compiled into oracle/_ref/libref_observations.so where the reference
                  sources exist; elsewhere the prebuilt library is used as it is"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import covis as CV
from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborb_oracle_observations.so")
_SRC = os.path.join(_HERE, "orb_oracle_observations.c")
_REF_SO = os.path.join(R._DIR, "libref_observations.so")
_REF_SRCS = [os.path.join(_HERE, "ref_shim", f) for f in ("ref_observations.cc", "ref_covis.cc")]
_lib = None
_ref_lib = None


def build(force=False):
    """Compile the oracle library, and the reference driver where the reference sources exist."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                               "-std=gnu11", "-shared", _SRC, "-o", _SO])
    root = R.REFERENCE_ROOT
    if os.path.isdir(os.path.join(root, "src")):
        base = R.build()
        if force or not os.path.exists(_REF_SO) or os.path.getmtime(_REF_SO) < max([os.path.getmtime(f) for f in _REF_SRCS] +
                                                                                   [os.path.getmtime(base)]):
            subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC",
                                   "-w", "-shared", "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"),
                                   "-I" + root, _REF_SRCS[0], "-o", _REF_SO, "-L" + R._DIR, "-lref_orbslam", "-Wl,-rpath,$ORIGIN",
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
        L.obs_oracle.argtypes = [i, vp, i, vp, vp, i, i, vp, vp, vp, i, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def observations(points, npoints, kf_mp, counts, cap, live, keys, ref_slot=None, obs_cap=None):
    """The entry's result on host arrays: (status, ptr, obs, nobs, ref_obs).  kf_mp [nframes*cap], counts / live / keys
    [nframes]; status 0, -1 (ORBFE_ERR_ARG) or -3 (ORBFE_ERR_CAPACITY) as the device reports it; obs is None unless 0, nobs
    None on -1, ref_obs None unless 0 with ref_slot given."""
    points = np.ascontiguousarray(points, np.int32)
    kf_mp, counts = np.ascontiguousarray(kf_mp, np.int32), np.ascontiguousarray(counts, np.int32)
    live, keys = np.ascontiguousarray(live, np.uint8), np.ascontiguousarray(keys, np.uint64)
    n, nframes = len(points), len(counts)
    if obs_cap is None:
        obs_cap = int(np.count_nonzero(kf_mp >= 0))
    ptr = np.zeros(n + 1, np.int32)
    obs = np.zeros(max(obs_cap, 1), np.int32)
    nobs = np.zeros(1, np.int32)
    rs = None if ref_slot is None else np.ascontiguousarray(ref_slot, np.int32)
    ro = None if ref_slot is None else np.zeros(max(n, 1), np.int32)
    rc = lib().obs_oracle(n, _p(points) if n else None, int(npoints), _p(kf_mp), _p(counts), nframes, int(cap), _p(live), _p(keys),
                          None if rs is None else _p(rs), int(obs_cap), _p(ptr), _p(obs), _p(nobs), None if ro is None else _p(ro))
    if rc != 0:
        return rc, ptr, None, (None if rc == -1 else int(nobs[0])), None
    return rc, ptr, obs[:ptr[-1]], int(nobs[0]), (None if ro is None else ro[:n])


def _ref():
    global _ref_lib
    if _ref_lib is None:
        if not os.path.exists(_REF_SO):
            build()
        L = C.CDLL(_REF_SO, mode=os.RTLD_NOW | os.RTLD_LOCAL)
        vp, i = C.c_void_p, C.c_int
        L.ref_cv_create.restype = vp
        L.ref_cv_free.argtypes = [vp]
        for f, a in (("ref_ob_add_keyframe", [vp, i]), ("ref_cv_add_point", [vp, i]), ("ref_cv_observe", [vp, i, i, i]),
                     ("ref_cv_update", [vp, i]), ("ref_cv_set_bad_keyframe", [vp, i]), ("ref_cv_set_bad_point", [vp, i]),
                     ("ref_cv_erase_match", [vp, i, i]), ("ref_cv_ordered", [vp, i, vp, vp, i]), ("ref_cv_weights", [vp, i, vp, vp, i]),
                     ("ref_cv_parent", [vp, i]), ("ref_cv_keyframe_bad", [vp, i]), ("ref_cv_matches", [vp, i, vp, i]),
                     ("ref_cv_observations", [vp, i, vp, vp, i]), ("ref_cv_point_bad", [vp, i]),
                     ("ref_ob_add_map_point", [vp, i, i, i]), ("ref_ob_add_observation", [vp, i, i, i]), ("ref_ob_replace", [vp, i, i]),
                     ("ref_ob_ba_erase", [vp, i, i]), ("ref_ob_reference", [vp, i])):
            getattr(L, f).argtypes = a
        L.ref_cv_observe_many.argtypes = [vp, i, vp, vp, vp]
        L.ref_ob_flatten.argtypes = [vp, i, vp, vp, i, vp, vp]
        L.ref_cv_add_points.argtypes = [vp, i, vp]
        L.ref_cv_keyframe_mnid.argtypes = [vp, i]
        L.ref_cv_keyframe_mnid.restype = C.c_long
        _ref_lib = L
    return _ref_lib


class RefObservations(CV.RefCovis):
    """RefCovis on libref_observations.so: keyframes with descriptors, and the edits Replace / BA erase / the halves of an
    observation, with GetReferenceKeyFrame() read back."""

    def __init__(self, cap=1 << 16):
        self.L = _ref()
        self.h = self.L.ref_cv_create()
        self._a, self._b = np.zeros(cap, np.int32), np.zeros(cap, np.int32)

    def add_keyframe(self, nfeatures):
        return self.L.ref_ob_add_keyframe(self.h, int(nfeatures))

    def add_map_point(self, kf, idx, mp):
        self.L.ref_ob_add_map_point(self.h, int(kf), int(idx), int(mp))

    def add_observation(self, mp, kf, idx):
        self.L.ref_ob_add_observation(self.h, int(mp), int(kf), int(idx))

    def replace(self, mp_from, mp_to):
        self.L.ref_ob_replace(self.h, int(mp_from), int(mp_to))

    def ba_erase(self, kf, mp):
        self.L.ref_ob_ba_erase(self.h, int(kf), int(mp))

    def reference(self, mp):
        return self.L.ref_ob_reference(self.h, int(mp))

    def flatten(self, points, slot_of, cap, ptr, obs):
        """the host build of the lists of `points` into ptr / obs (int32 arrays, preallocated); returns the total"""
        return self.L.ref_ob_flatten(self.h, len(points), _p(points), _p(slot_of), int(cap), _p(ptr), _p(obs))
