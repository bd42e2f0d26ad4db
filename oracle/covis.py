"""The covisibility graph (KeyFrame::UpdateConnections and its helpers, src/KeyFrame.cc) for the tests of orbfe_covis_*
(TEST INFRASTRUCTURE ONLY).

  CovisOracle   the oracle's restatement, oracle/orb_oracle_covis.c in oracle/liborb_oracle.so; replay() runs a batch as
                consecutive calls
  RefCovis      the reference's own KeyFrame / MapPoint on a scripted map: oracle/ref_shim/ref_covis.cc (through
                ref_observations.cc) in oracle/_ref/libref_drivers.so, linked against libref_orbslam.so (the reference's
                sources, unmodified)

REF_CV is the signature table of the ref_cv_* driver functions; oracle.observations, oracle.kf_culling and oracle.local_map
extend it for the libraries that hold those functions too."""
import ctypes as C

import numpy as np

from . import _cdll
from ._cdll import p as _p

vp, i = C.c_void_p, C.c_int
lib = _cdll.loader("liborb_oracle.so", {
    "covis_oracle_create": (vp, [i]),
    "covis_oracle_free": (None, [vp]),
    "covis_oracle_add": (None, [vp, i, i, C.c_uint64]),
    "covis_oracle_update": (i, [vp, i, vp, vp, i, vp, vp]),
    "covis_oracle_erase": (None, [vp, i]),
    "covis_oracle_clear": (None, [vp]),
    "covis_oracle_ordered": (i, [vp, i, vp, vp]),
    "covis_oracle_weights": (i, [vp, i, vp, vp]),
    "covis_oracle_parent": (i, [vp, i]),
    "covis_oracle_live": (i, [vp, i]),
})
REF_CV = {
    "ref_cv_create": (vp, []),
    "ref_cv_free": (i, [vp]),
    "ref_cv_set_kf_order": (i, [vp, i, vp]),
    "ref_cv_add_keyframe": (i, [vp, i]),
    "ref_cv_add_point": (i, [vp, i]),
    "ref_cv_add_points": (i, [vp, i, vp]),
    "ref_cv_observe": (i, [vp, i, i, i]),
    "ref_cv_observe_many": (i, [vp, i, vp, vp, vp]),
    "ref_cv_update": (i, [vp, i]),
    "ref_cv_set_bad_keyframe": (i, [vp, i]),
    "ref_cv_set_bad_point": (i, [vp, i]),
    "ref_cv_erase_match": (i, [vp, i, i]),
    "ref_cv_ordered": (i, [vp, i, vp, vp, i]),
    "ref_cv_weights": (i, [vp, i, vp, vp, i]),
    "ref_cv_parent": (i, [vp, i]),
    "ref_cv_keyframe_bad": (i, [vp, i]),
    "ref_cv_keyframe_mnid": (C.c_long, [vp, i]),
    "ref_cv_matches": (i, [vp, i, vp, i]),
    "ref_cv_observations": (i, [vp, i, vp, vp, i]),
    "ref_cv_point_bad": (i, [vp, i]),
}
# newer than the rest of the driver: a prebuilt library may lack it (see ref_kf_order_available)
REF_CV_OPTIONAL = ("ref_cv_set_kf_order",)
_ref = _cdll.loader("_ref/libref_drivers.so", REF_CV, REF_CV_OPTIONAL)


def ref_available():
    return _cdll.ref_available("libref_drivers.so")


def ref_kf_order_available():
    """the driver is built and can lay keyframes out in a given order (RefCovis.set_kf_order)"""
    return ref_available() and _cdll.has(_ref, "ref_cv_set_kf_order")


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


class RefCovis:
    """A scripted map of the reference's own KeyFrames and MapPoints (ids = creation order; the first keyframe has mnId 0).
    Pointer order is creation order unless set_kf_order() gives another."""

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

    def set_kf_order(self, rank):
        """Before the first keyframe: keyframe k is placed at rank[k] among the keyframes' addresses (rank a permutation of
        0 .. n-1), so every pointer order of the map is rank order rather than creation order; at most n keyframes follow."""
        r = np.ascontiguousarray(rank, np.int32)
        if self.L.ref_cv_set_kf_order(self.h, len(r), _p(r)) != 0:
            raise ValueError("ref_cv_set_kf_order: a keyframe exists or rank is not a permutation")

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
