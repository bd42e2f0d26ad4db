"""LocalMapping::KeyFrameCulling with SetBadFlag's map-point half on the keyframes' rows, for the tests of
orbfe_covis_keyframe_culling_device (TEST INFRASTRUCTURE ONLY).

  cull()          the oracle's restatement, oracle/orb_oracle_kf_culling.c in oracle/liborb_oracle.so
  RefKfCulling    oracle.observations.RefObservations plus keypoint octaves, mbNotErase and the reference's own
                  LocalMapping::KeyFrameCulling: oracle/ref_shim/ref_kf_culling.cc and the reference's src/LocalMapping.cc,
                  compiled against the stand-in headers of oracle/ref_shim_slam/ into oracle/_ref/libref_kf_culling.so"""
import ctypes as C

import numpy as np

from . import _cdll
from . import covis as CV
from . import observations as OB
from ._cdll import p as _p

vp, i = C.c_void_p, C.c_int
lib = _cdll.loader("liborb_oracle.so", {
    "kfc_oracle": (i, [i, vp, vp, vp, vp, vp, vp, vp, vp, i, i, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp])})
_ref = _cdll.loader("_ref/libref_kf_culling.so", {
    **OB.REF_OB,
    "ref_kc_set_octaves": (i, [vp, i, i, vp]),
    "ref_kc_set_not_erase": (i, [vp, i]),
    "ref_kc_cull": (i, [vp, i, vp, vp, i, vp]),
}, CV.REF_CV_OPTIONAL)

# verdicts (ORBFE_CULL_*)
KEPT, SKIP_ID0, ERASED, NOT_ERASE, RETIRED = 0, 1, 2, 3, 4


def ref_available():
    return _cdll.ref_available("libref_kf_culling.so")


def ref_kf_order_available():
    """the driver is built and can lay keyframes out in a given order (RefCovis.set_kf_order)"""
    return ref_available() and _cdll.has(_ref, "ref_cv_set_kf_order")


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
