"""LocalMapping::KeyFrameCulling with SetBadFlag's map-point half on the keyframes' rows, for the tests of
orbfe_covis_keyframe_culling_device (TEST INFRASTRUCTURE ONLY).

  cull()          the oracle's restatement, oracle/orb_oracle_kf_culling.c, compiled here into oracle/liborb_oracle_kf_culling.so
                  with the flags of oracle/Makefile
  RefKfCulling    oracle.observations.RefObservations plus keypoint octaves, mbNotErase and the reference's own
                  LocalMapping::KeyFrameCulling: oracle/ref_shim/ref_kf_culling.cc and the reference's src/LocalMapping.cc,
                  compiled against the stand-in headers of oracle/ref_shim_lm/ into oracle/_ref/libref_kf_culling.so where the
                  reference sources exist; elsewhere the prebuilt library is used as it is"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import observations as OB
from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborb_oracle_kf_culling.so")
_SRC = os.path.join(_HERE, "orb_oracle_kf_culling.c")
_REF_SO = os.path.join(R._DIR, "libref_kf_culling.so")
_LM_OBJ = os.path.join(R._DIR, "obj", "LocalMapping_kf_culling.o")
_SHIM_LM = os.path.join(_HERE, "ref_shim_lm")
_REF_SRCS = [os.path.join(_HERE, "ref_shim", f) for f in ("ref_kf_culling.cc", "ref_observations.cc", "ref_covis.cc")] + \
    [os.path.join(dp, f) for dp, _, fs in os.walk(_SHIM_LM) for f in fs]
_lib = None
_ref_lib = None

# verdicts (ORBFE_CULL_*)
KEPT, SKIP_ID0, ERASED, NOT_ERASE, RETIRED = 0, 1, 2, 3, 4


def build(force=False):
    """Compile the oracle library, and the reference driver where the reference sources exist."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                               "-std=gnu11", "-shared", _SRC, "-o", _SO])
    root = R.REFERENCE_ROOT
    if os.path.isdir(os.path.join(root, "src")):
        base = R.build()
        lm_src = os.path.join(root, "src", "LocalMapping.cc")
        newest = max([os.path.getmtime(f) for f in _REF_SRCS] + [os.path.getmtime(base), os.path.getmtime(lm_src)])
        if force or not os.path.exists(_REF_SO) or os.path.getmtime(_REF_SO) < newest:
            flags = ["-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-w", "-I" + _SHIM_LM,
                     "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"), "-I" + root]
            os.makedirs(os.path.dirname(_LM_OBJ), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++"] + flags + ["-include", os.path.join(_SHIM_LM, "ref_lm_prelude.h"), "-c", lm_src,
                                                              "-o", _LM_OBJ])
            subprocess.check_call(["/usr/bin/g++"] + flags + ["-shared", _REF_SRCS[0], _LM_OBJ, "-o", _REF_SO, "-L" + R._DIR,
                                                              "-lref_orbslam", "-Wl,-rpath,$ORIGIN", "-lpthread"])
    return _SO


def ref_available():
    return os.path.exists(_REF_SO) and R.available()


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, i = C.c_void_p, C.c_int
        L.kfc_oracle.argtypes = [i, vp, vp, vp, vp, vp, vp, vp, vp, i, i, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cull(cand, live, id0, keys, not_erase, kf_mp, counts, octave, cap, point_bad, ref_slot, obs_cap=None):
    """The entry's result on host arrays (cand = the current keyframe's ordered list as slots; live / id0 / keys / not_erase
    per slot; kf_mp and octave [nframes*cap]).  Returns a dict: status (0, -1, -3), nobs (None on -1) and, on 0, verdict_slot,
    verdict, nmps, nred, bad_points and the updated kf_mp, point_bad, ref_slot (the inputs are not changed)."""
    cand = np.ascontiguousarray(cand, np.int32)
    counts = np.ascontiguousarray(counts, np.int32)
    nframes, npoints = len(counts), len(point_bad)
    kf_mp = np.array(kf_mp, np.int32).ravel()
    octave = np.ascontiguousarray(octave, np.int32).ravel()
    live, id0, ne = (np.ascontiguousarray(x, np.uint8) for x in (live, id0, not_erase))
    keys = np.ascontiguousarray(keys, np.uint64)
    pb, rs = np.array(point_bad, np.uint8), np.array(ref_slot, np.int32)
    if obs_cap is None:
        obs_cap = int(np.count_nonzero(kf_mp >= 0))
    n = len(cand)
    vs, vd, nm, nr = (np.zeros(max(n, 1), np.int32) for _ in range(4))
    bp = np.zeros(max(npoints, 1), np.int32)
    nobs, nbad = np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = lib().kfc_oracle(n, _p(cand), _p(live), _p(id0), _p(keys), _p(ne), _p(kf_mp), _p(counts), _p(octave), nframes, int(cap),
                          _p(pb), _p(rs), npoints, int(obs_cap), _p(nobs), _p(vs), _p(vd), _p(nm), _p(nr), _p(bp), _p(nbad))
    out = dict(status=rc, nobs=None if rc == -1 else int(nobs[0]))
    if rc == 0:
        out.update(verdict_slot=vs[:n], verdict=vd[:n], nmps=nm[:n], nred=nr[:n], bad_points=bp[:int(nbad[0])], kf_mp=kf_mp,
                   point_bad=pb, ref_slot=rs)
    return out


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
                     ("ref_ob_ba_erase", [vp, i, i]), ("ref_ob_reference", [vp, i]), ("ref_kc_set_octaves", [vp, i, i, vp]),
                     ("ref_kc_set_not_erase", [vp, i]), ("ref_kc_cull", [vp, i, vp, vp, i, vp])):
            getattr(L, f).argtypes = a
        L.ref_cv_observe_many.argtypes = [vp, i, vp, vp, vp]
        L.ref_ob_flatten.argtypes = [vp, i, vp, vp, i, vp, vp]
        L.ref_cv_add_points.argtypes = [vp, i, vp]
        L.ref_cv_keyframe_mnid.argtypes = [vp, i]
        L.ref_cv_keyframe_mnid.restype = C.c_long
        _ref_lib = L
    return _ref_lib


class RefKfCulling(OB.RefObservations):
    """RefObservations on libref_kf_culling.so, with keypoint octaves, mbNotErase and KeyFrameCulling()."""

    def __init__(self, cap=1 << 16):
        self.L = _ref()
        self.h = self.L.ref_cv_create()
        self._a, self._b = np.zeros(cap, np.int32), np.zeros(cap, np.int32)

    def set_octaves(self, kf, octaves):
        o = np.ascontiguousarray(octaves, np.int32)
        self.L.ref_kc_set_octaves(self.h, int(kf), len(o), _p(o))

    def set_not_erase(self, kf):
        self.L.ref_kc_set_not_erase(self.h, int(kf))

    def cull(self, current):
        """KeyFrameCulling() with `current` as mpCurrentKeyFrame: (keyframe ids of the list, verdicts, nanoseconds)"""
        ns = np.zeros(1, np.int64)
        n = self.L.ref_kc_cull(self.h, int(current), _p(self._a), _p(self._b), len(self._a), _p(ns))
        assert n <= len(self._a)
        return self._a[:n].tolist(), self._b[:n].tolist(), int(ns[0])
