"""Tracking::UpdateReference (UpdateReferenceKeyFrames and UpdateReferencePoints) on the keyframes' rows and the covisibility
graph, for the tests of orbfe_covis_local_map_device (TEST INFRASTRUCTURE ONLY).

  local_map()   the oracle's restatement, oracle/orb_oracle_local_map.c in oracle/liborb_oracle.so
  RefLocalMap   oracle.observations.RefObservations plus the reference's own Tracking::UpdateReference:
                oracle/ref_shim/ref_local_map.cc and the reference's src/Tracking.cc, compiled against the stand-in headers of
                oracle/ref_shim_slam/ into oracle/_ref/libref_local_map.so"""
import ctypes as C

import numpy as np

from . import _cdll
from . import covis as CV
from . import observations as OB
from ._cdll import p as _p

NEIGH = 10   # GetBestCovisibilityKeyFrames(10)
vp, i = C.c_void_p, C.c_int
lib = _cdll.loader("liborb_oracle.so", {"lm_oracle": (i, [i, vp, vp, i, vp, vp, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp])})
_ref = _cdll.loader("_ref/libref_local_map.so", {
    **OB.REF_OB,
    "ref_lm_free": (i, [vp]),
    "ref_lm_to_be_erased": (i, [vp, i]),
    "ref_lm_update_reference": (i, [vp, i, vp, vp, i, vp, vp, i, vp, vp]),
}, CV.REF_CV_OPTIONAL)


def ref_available():
    return _cdll.ref_available("libref_local_map.so")


def ref_kf_order_available():
    """the driver is built and can lay keyframes out in a given order (RefCovis.set_kf_order)"""
    return ref_available() and _cdll.has(_ref, "ref_cv_set_kf_order")


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
