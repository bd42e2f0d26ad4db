"""ORBVocabulary::score and LoopClosing::DetectLoop's minScore loop (src/LoopClosing.cc:117-131) for the tests of
orbfe_bow_min_score_device / orbfe_bow_score (TEST INFRASTRUCTURE ONLY).

  bow_score, loop_min_score   the oracle's restatement, oracle/orb_oracle_bow_score.c in oracle/liborb_oracle.so
  RefVocabularyScore          the reference's own ORBVocabulary::score: oracle/ref_shim/ref_voc_score.cc in
                              oracle/_ref/libref_drivers.so, linked against libref_orbslam.so (the reference's DBoW2,
                              unmodified)"""
import ctypes as C

import numpy as np

from . import _cdll
from ._cdll import p as _p

vp, i = C.c_void_p, C.c_int
lib = _cdll.loader("liborb_oracle.so", {
    "orb_oracle_bow_score": (C.c_double, [vp, vp, i, vp, vp, i]),
    "orb_oracle_loop_min_score": (C.c_float, [vp, vp, i, i, vp, vp, vp, vp]),
})
_ref = _cdll.loader("_ref/libref_drivers.so", {
    "ref_voc_score_create": (vp, [C.c_char_p]),
    "ref_voc_score_free": (None, [vp]),
    "ref_voc_score": (C.c_double, [vp, vp, vp, i, vp, vp, i]),
})


def ref_available():
    return _cdll.ref_available("libref_drivers.so")


def _bow(ids, vals):
    return np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(vals, np.float64)


def bow_score(ids1, vals1, ids2, vals2):
    """L1Scoring::score of two BowVectors (word ids ascending), the double ORBVocabulary::score returns."""
    (i1, v1), (i2, v2) = _bow(ids1, vals1), _bow(ids2, vals2)
    return lib().orb_oracle_bow_score(_p(i1), _p(v1), len(i1), _p(i2), _p(v2), len(i2))


def loop_min_score(q_ids, q_vals, covisibles, bad=None):
    """minScore of LoopClosing::DetectLoop as a numpy float32: covisibles = [(ids, vals), ...] in the order of
    GetVectorCovisibleKeyFrames(), bad[k] true for a keyframe with isBad()."""
    qi, qv = _bow(q_ids, q_vals)
    n = len(covisibles)
    ptr = np.cumsum([0] + [len(c[0]) for c in covisibles]).astype(np.int32)
    ci, cv = _bow(np.concatenate([np.asarray(c[0], np.int32) for c in covisibles] + [np.zeros(1, np.int32)]),
                  np.concatenate([np.asarray(c[1], np.float64) for c in covisibles] + [np.zeros(1)]))
    flags = np.zeros(n + 1, np.uint8)
    if bad is not None:
        flags[:n] = np.asarray(bad, bool)
    return np.float32(lib().orb_oracle_loop_min_score(_p(qi), _p(qv), len(qi), n, _p(ptr), _p(ci), _p(cv), _p(flags)))


class RefVocabularyScore:
    """score() of a reference ORBVocabulary loaded from DBoW2's text format."""

    def __init__(self, vocabulary_text_path):
        self.L = _ref()
        self.h = self.L.ref_voc_score_create(vocabulary_text_path.encode())
        assert self.h, "loadFromTextFile failed"

    def score(self, ids1, vals1, ids2, vals2):
        (i1, v1), (i2, v2) = _bow(ids1, vals1), _bow(ids2, vals2)
        return self.L.ref_voc_score(self.h, _p(i1), _p(v1), len(i1), _p(i2), _p(v2), len(i2))

    def close(self):
        if self.h:
            self.L.ref_voc_score_free(self.h)
            self.h = None
