"""The covisibility graph (KeyFrame::UpdateConnections and its helpers, src/KeyFrame.cc) for the tests of orbfe_covis_*
(TEST INFRASTRUCTURE ONLY).

  CovisOracle   the oracle's restatement, oracle/orb_oracle_covis.c, compiled here into oracle/liborb_oracle_covis.so with
                the flags of oracle/Makefile; replay() runs a batch as consecutive calls
  RefCovis      the reference's own KeyFrame / MapPoint on a scripted map: oracle/ref_shim/ref_covis.cc compiled into
                oracle/_ref/libref_covis.so, linked against libref_orbslam.so (the reference's sources, unmodified), where
                the reference sources exist; elsewhere the prebuilt library is used as it is"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import ref as R

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborb_oracle_covis.so")
_SRC = os.path.join(_HERE, "orb_oracle_covis.c")
_REF_SO = os.path.join(R._DIR, "libref_covis.so")
_REF_SRC = os.path.join(_HERE, "ref_shim", "ref_covis.cc")
_lib = None
_ref_lib = None


def build(force=False):
    """Compile the oracle library, and the reference driver where the reference sources exist (after `make ref`)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["/usr/bin/gcc", "-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-Wall",
                               "-std=gnu11", "-shared", _SRC, "-o", _SO])
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
        L.covis_oracle_create.argtypes = [i]
        L.covis_oracle_create.restype = vp
        L.covis_oracle_free.argtypes = [vp]
        L.covis_oracle_free.restype = None
        L.covis_oracle_add.argtypes = [vp, i, i, C.c_uint64]
        L.covis_oracle_add.restype = None
        L.covis_oracle_update.argtypes = [vp, i, vp, vp, i, vp, vp]
        L.covis_oracle_erase.argtypes = [vp, i]
        L.covis_oracle_erase.restype = None
        L.covis_oracle_clear.argtypes = [vp]
        L.covis_oracle_clear.restype = None
        L.covis_oracle_ordered.argtypes = [vp, i, vp, vp]
        L.covis_oracle_weights.argtypes = [vp, i, vp, vp]
        L.covis_oracle_parent.argtypes = [vp, i]
        L.covis_oracle_live.argtypes = [vp, i]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class CovisOracle:
    """The oracle's graph over K slots.  Inputs of update() are those of orbfe_covis_update_connections_device as host
    arrays: kf_mp [K*cap], counts [K], group_ptr, obs."""

    def __init__(self, K):
        self.L, self.K = lib(), int(K)
        self.h = self.L.covis_oracle_create(self.K)
        self._s, self._w = np.zeros(self.K, np.int32), np.zeros(self.K, np.int32)

    def close(self):
        if self.h:
            self.L.covis_oracle_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, slot, id_, key):
        self.L.covis_oracle_add(self.h, int(slot), int(id_), int(key))

    def update(self, slot, kf_mp, counts, cap, group_ptr, obs):
        """UpdateConnections of one slot; returns the parent it set, else -1."""
        return self.L.covis_oracle_update(self.h, int(slot), _p(kf_mp), _p(counts), int(cap), _p(group_ptr), _p(obs))

    def replay(self, slots, kf_mp, counts, cap, group_ptr, obs):
        """A batch as consecutive calls in order; returns the parents."""
        kf_mp, counts = np.ascontiguousarray(kf_mp, np.int32), np.ascontiguousarray(counts, np.int32)
        group_ptr = np.ascontiguousarray(group_ptr, np.int32)
        obs = np.ascontiguousarray(obs if len(obs) else [0], np.int32)
        return [self.update(s, kf_mp, counts, cap, group_ptr, obs) for s in slots]

    def erase(self, slot):
        self.L.covis_oracle_erase(self.h, int(slot))

    def clear(self):
        self.L.covis_oracle_clear(self.h)

    def ordered(self, slot):
        """(slots, weights) of the ordered list."""
        n = self.L.covis_oracle_ordered(self.h, int(slot), _p(self._s), _p(self._w))
        return self._s[:n].tolist(), self._w[:n].tolist()

    def weights(self, slot):
        """(slots, weights) of the weight map in key order."""
        n = self.L.covis_oracle_weights(self.h, int(slot), _p(self._s), _p(self._w))
        return self._s[:n].tolist(), self._w[:n].tolist()

    def parent(self, slot):
        return self.L.covis_oracle_parent(self.h, int(slot))

    def live(self, slot):
        return bool(self.L.covis_oracle_live(self.h, int(slot)))


def _ref():
    global _ref_lib
    if _ref_lib is None:
        if not os.path.exists(_REF_SO):
            build()
        L = C.CDLL(_REF_SO, mode=os.RTLD_NOW | os.RTLD_LOCAL)
        vp, i = C.c_void_p, C.c_int
        L.ref_cv_create.restype = vp
        L.ref_cv_free.argtypes = [vp]
        for f, a in (("ref_cv_add_keyframe", [vp, i]), ("ref_cv_add_point", [vp, i]), ("ref_cv_observe", [vp, i, i, i]),
                     ("ref_cv_update", [vp, i]), ("ref_cv_set_bad_keyframe", [vp, i]), ("ref_cv_set_bad_point", [vp, i]),
                     ("ref_cv_erase_match", [vp, i, i]), ("ref_cv_ordered", [vp, i, vp, vp, i]), ("ref_cv_weights", [vp, i, vp, vp, i]),
                     ("ref_cv_parent", [vp, i]), ("ref_cv_keyframe_bad", [vp, i]), ("ref_cv_matches", [vp, i, vp, i]),
                     ("ref_cv_observations", [vp, i, vp, vp, i]), ("ref_cv_point_bad", [vp, i])):
            getattr(L, f).argtypes = a
        L.ref_cv_observe_many.argtypes = [vp, i, vp, vp, vp]
        L.ref_cv_add_points.argtypes = [vp, i, vp]
        L.ref_cv_keyframe_mnid.argtypes = [vp, i]
        L.ref_cv_keyframe_mnid.restype = C.c_long
        _ref_lib = L
    return _ref_lib


class RefCovis:
    """A scripted map of the reference's own KeyFrames and MapPoints (ids = creation order; the first keyframe has mnId 0)."""

    def __init__(self, cap=1 << 16):
        self.L = _ref()
        self.h = self.L.ref_cv_create()
        self._a, self._b = np.zeros(cap, np.int32), np.zeros(cap, np.int32)

    def close(self):
        if self.h:
            self.L.ref_cv_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_keyframe(self, nfeatures):
        return self.L.ref_cv_add_keyframe(self.h, int(nfeatures))

    def add_point(self, ref_kf):
        return self.L.ref_cv_add_point(self.h, int(ref_kf))

    def observe(self, mp, kf, idx):
        self.L.ref_cv_observe(self.h, int(mp), int(kf), int(idx))

    def add_points(self, ref_kfs):
        r = np.ascontiguousarray(ref_kfs, np.int32)
        return self.L.ref_cv_add_points(self.h, len(r), _p(r))

    def observe_many(self, mp, kf, idx):
        mp, kf, idx = (np.ascontiguousarray(x, np.int32) for x in (mp, kf, idx))
        self.L.ref_cv_observe_many(self.h, len(mp), _p(mp), _p(kf), _p(idx))

    def update(self, kf):
        self.L.ref_cv_update(self.h, int(kf))

    def set_bad_keyframe(self, kf):
        self.L.ref_cv_set_bad_keyframe(self.h, int(kf))

    def set_bad_point(self, mp):
        self.L.ref_cv_set_bad_point(self.h, int(mp))

    def erase_match(self, kf, idx):
        self.L.ref_cv_erase_match(self.h, int(kf), int(idx))

    def _pair(self, fn, x):
        n = fn(self.h, int(x), _p(self._a), _p(self._b), len(self._a))
        assert n <= len(self._a)
        return self._a[:n].tolist(), self._b[:n].tolist()

    def ordered(self, kf):
        return self._pair(self.L.ref_cv_ordered, kf)

    def weights(self, kf):
        return self._pair(self.L.ref_cv_weights, kf)

    def observations(self, mp):
        return self._pair(self.L.ref_cv_observations, mp)

    def parent(self, kf):
        return self.L.ref_cv_parent(self.h, int(kf))

    def keyframe_bad(self, kf):
        return bool(self.L.ref_cv_keyframe_bad(self.h, int(kf)))

    def mnid(self, kf):
        return self.L.ref_cv_keyframe_mnid(self.h, int(kf))

    def matches(self, kf):
        n = self.L.ref_cv_matches(self.h, int(kf), _p(self._a), len(self._a))
        return self._a[:n].tolist()

    def point_bad(self, mp):
        return bool(self.L.ref_cv_point_bad(self.h, int(mp)))
