"""Tracking::UpdateReference (UpdateReferenceKeyFrames and UpdateReferencePoints) on the keyframes' rows and the covisibility
graph, for the tests of orbfe_covis_local_map_device (TEST INFRASTRUCTURE ONLY).

  local_map()   the oracle's restatement, oracle/orb_oracle_local_map.c, compiled here into oracle/liborb_oracle_local_map.so
                with the flags of oracle/Makefile
  RefLocalMap   oracle.observations.RefObservations plus the reference's own Tracking::UpdateReference:
                oracle/ref_shim/ref_local_map.cc and the reference's src/Tracking.cc, compiled against the stand-in headers of
                oracle/ref_shim_tr/ and oracle/ref_shim_lm/ into oracle/_ref/libref_local_map.so where the reference sources
                exist; elsewhere the prebuilt library is used as it is"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import observations as OB
from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborb_oracle_local_map.so")
_SRC = os.path.join(_HERE, "orb_oracle_local_map.c")
_REF_SO = os.path.join(R._DIR, "libref_local_map.so")
_TR_OBJ = os.path.join(R._DIR, "obj", "Tracking_local_map.o")
_SHIM_LM = os.path.join(_HERE, "ref_shim_lm")
_SHIM_TR = os.path.join(_HERE, "ref_shim_tr")
_REF_SRCS = [os.path.join(_HERE, "ref_shim", f) for f in ("ref_local_map.cc", "ref_observations.cc", "ref_covis.cc")] + \
    [os.path.join(dp, f) for d in (_SHIM_LM, _SHIM_TR) for dp, _, fs in os.walk(d) for f in fs]
NEIGH = 10   # GetBestCovisibilityKeyFrames(10)
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
        tr_src = os.path.join(root, "src", "Tracking.cc")
        newest = max([os.path.getmtime(f) for f in _REF_SRCS] + [os.path.getmtime(base), os.path.getmtime(tr_src)])
        if force or not os.path.exists(_REF_SO) or os.path.getmtime(_REF_SO) < newest:
            flags = ["-std=c++14", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-w", "-I" + _SHIM_TR,
                     "-I" + _SHIM_LM, "-I" + os.path.join(_HERE, "ref_shim"), "-I" + os.path.join(root, "include"), "-I" + root]
            os.makedirs(os.path.dirname(_TR_OBJ), exist_ok=True)
            subprocess.check_call(["/usr/bin/g++"] + flags + ["-include", os.path.join(_SHIM_LM, "ref_lm_prelude.h"), "-include",
                                                              os.path.join(_SHIM_TR, "ref_tr_prelude.h"), "-c", tr_src, "-o", _TR_OBJ])
            subprocess.check_call(["/usr/bin/g++"] + flags + ["-shared", _REF_SRCS[0], _TR_OBJ, "-o", _REF_SO, "-L" + R._DIR,
                                                              "-lref_orbslam", "-Wl,-rpath,$ORIGIN", "-Wl,-z,defs", "-lpthread"])
    return _SO


def ref_available():
    return os.path.exists(_REF_SO) and R.available()


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, i = C.c_void_p, C.c_int
        L.lm_oracle.argtypes = [i, vp, vp, i, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def neighbours(lists, nframes):
    """(nb [nframes*NEIGH], nnb [nframes]) from {slot: its ordered list as the graph holds it}"""
    nb = np.full((nframes, NEIGH), -1, np.int32)
    nnb = np.zeros(nframes, np.int32)
    for s, lst in lists.items():
        lst = list(lst)[:NEIGH]
        nb[s, :len(lst)] = lst
        nnb[s] = len(lst)
    return nb.ravel(), nnb


def local_map(frame_mp, point_bad, kf_mp, counts, cap, live, keys, nb, nnb):
    """The entry's result on host arrays (kf_mp [nframes*cap]; counts / live / keys [nframes]; nb / nnb from neighbours()).
    Returns a dict: status (0 or -1) and, on 0, frame_mp (the cells afterwards), local_kf, ref_kf and local_points (the
    inputs are not changed)."""
    fm = np.array(frame_mp, np.int32).ravel()
    pb = np.ascontiguousarray(point_bad, np.uint8)
    kf_mp, counts = np.ascontiguousarray(kf_mp, np.int32).ravel(), np.ascontiguousarray(counts, np.int32)
    live, keys = np.ascontiguousarray(live, np.uint8), np.ascontiguousarray(keys, np.uint64)
    nb, nnb = np.ascontiguousarray(nb, np.int32), np.ascontiguousarray(nnb, np.int32)
    nframes, npoints = len(counts), len(pb)
    lk, lp = np.zeros(max(nframes, 1), np.int32), np.zeros(max(npoints, 1), np.int32)
    nlk, ref, nlp = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32)
    rc = lib().lm_oracle(len(fm), _p(fm) if len(fm) else None, _p(pb) if npoints else None, npoints, _p(kf_mp), _p(counts), nframes,
                         int(cap), _p(live), _p(keys), _p(nb), _p(nnb), _p(lk), _p(nlk), _p(ref), _p(lp), _p(nlp))
    out = dict(status=rc)
    if rc == 0:
        out.update(frame_mp=fm, local_kf=lk[:int(nlk[0])], ref_kf=int(ref[0]), local_points=lp[:int(nlp[0])])
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
        L.ref_lm_free.argtypes = [vp]
        for f, a in (("ref_ob_add_keyframe", [vp, i]), ("ref_cv_add_point", [vp, i]), ("ref_cv_observe", [vp, i, i, i]),
                     ("ref_cv_update", [vp, i]), ("ref_cv_set_bad_keyframe", [vp, i]), ("ref_cv_set_bad_point", [vp, i]),
                     ("ref_cv_erase_match", [vp, i, i]), ("ref_cv_ordered", [vp, i, vp, vp, i]), ("ref_cv_weights", [vp, i, vp, vp, i]),
                     ("ref_cv_parent", [vp, i]), ("ref_cv_keyframe_bad", [vp, i]), ("ref_cv_matches", [vp, i, vp, i]),
                     ("ref_cv_observations", [vp, i, vp, vp, i]), ("ref_cv_point_bad", [vp, i]),
                     ("ref_ob_add_map_point", [vp, i, i, i]), ("ref_ob_add_observation", [vp, i, i, i]), ("ref_ob_replace", [vp, i, i]),
                     ("ref_ob_ba_erase", [vp, i, i]), ("ref_ob_reference", [vp, i]), ("ref_lm_to_be_erased", [vp, i]),
                     ("ref_lm_update_reference", [vp, i, vp, vp, i, vp, vp, i, vp, vp])):
            getattr(L, f).argtypes = a
        L.ref_cv_observe_many.argtypes = [vp, i, vp, vp, vp]
        L.ref_ob_flatten.argtypes = [vp, i, vp, vp, i, vp, vp]
        L.ref_cv_add_points.argtypes = [vp, i, vp]
        L.ref_cv_keyframe_mnid.argtypes = [vp, i]
        L.ref_cv_keyframe_mnid.restype = C.c_long
        _ref_lib = L
    return _ref_lib


class RefLocalMap(OB.RefObservations):
    """RefObservations on libref_local_map.so, with mbToBeErased and Tracking::UpdateReference()."""

    def __init__(self, cap=1 << 16):
        self.L = _ref()
        self.h = self.L.ref_cv_create()
        self._a, self._b = np.zeros(cap, np.int32), np.zeros(cap, np.int32)

    def close(self):
        if self.h:
            self.L.ref_lm_free(self.h)
            self.h = None

    def to_be_erased(self, kf):
        self.L.ref_lm_to_be_erased(self.h, int(kf))

    def update_reference(self, frame_mp):
        """UpdateReference() for a frame whose mvpMapPoints are frame_mp (point indices, -1 = NULL): (the frame's cells
        afterwards, mvpLocalKeyFrames as creation indices, mpReferenceKF (-1 for NULL), mvpLocalMapPoints, nanoseconds)"""
        fm = np.array(frame_mp, np.int32).ravel()
        lk = np.zeros(1 << 16, np.int32)
        lp = np.zeros(max(len(self._a), 1), np.int32)
        ref, nlp, ns = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int64)
        nlk = self.L.ref_lm_update_reference(self.h, len(fm), _p(fm) if len(fm) else None, _p(lk), len(lk), _p(ref), _p(lp), len(lp),
                                             _p(nlp), _p(ns))
        assert nlk <= len(lk) and int(nlp[0]) <= len(lp)
        return fm, lk[:nlk].tolist(), int(ref[0]), lp[:int(nlp[0])].tolist(), int(ns[0])
