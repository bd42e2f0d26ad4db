"""MapPoint::GetObservations() of named points as the inverse of the live keyframes' rows, for the tests of
orbfe_covis_observations_device (TEST INFRASTRUCTURE ONLY).

  observations()  the oracle's restatement, oracle/orb_oracle_observations.c in oracle/liborb_oracle.so
  RefObservations the reference's own KeyFrame / MapPoint on a scripted map (oracle.covis.RefCovis) plus MapPoint::Replace,
                  the local-BA outlier erase, the halves of an observation and GetReferenceKeyFrame():
                  oracle/ref_shim/ref_observations.cc in oracle/_ref/libref_drivers.so

REF_OB is oracle.covis.REF_CV plus the ref_ob_* functions; oracle.kf_culling and oracle.local_map extend it."""
import ctypes as C

import numpy as np

from . import _cdll
from . import covis as CV
from ._cdll import p as _p

vp, i = C.c_void_p, C.c_int
lib = _cdll.loader("liborb_oracle.so", {"obs_oracle": (i, [i, vp, i, vp, vp, i, i, vp, vp, vp, i, vp, vp, vp, vp])})
REF_OB = {
    **CV.REF_CV,
    "ref_ob_add_keyframe": (i, [vp, i]),
    "ref_ob_add_map_point": (i, [vp, i, i, i]),
    "ref_ob_add_observation": (i, [vp, i, i, i]),
    "ref_ob_replace": (i, [vp, i, i]),
    "ref_ob_ba_erase": (i, [vp, i, i]),
    "ref_ob_reference": (i, [vp, i]),
    "ref_ob_flatten": (i, [vp, i, vp, vp, i, vp, vp]),
}
_ref = _cdll.loader("_ref/libref_drivers.so", REF_OB, CV.REF_CV_OPTIONAL)
ref_available = CV.ref_available


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


class RefObservations(CV.RefCovis):
    """RefCovis with the ref_ob_* driver functions: keyframes with descriptors, and the edits Replace / BA erase / the halves of an
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
